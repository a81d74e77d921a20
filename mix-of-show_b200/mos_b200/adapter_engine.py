"""AdapterEngine — the T2I-Adapter network (diffusers 0.19.3 `T2IAdapter`, adapter_type 'full_adapter') on the GPU, built
only from libmos_sm100 kernels.  Owns the call the reference makes once per image:

    keypose_adapter_state = self.keypose_adapter(keypose_input)      mixofshow/pipelines/pipeline_regionally_t2iadapter.py:474-482

Topology (state-dict names `adapter.*`):
    x = PixelUnshuffle(8)(image); x = conv_in(x)                               3x3, Cin*64 -> channels[0]
    level l: [AvgPool2d(2) if l > 0] [in_conv 1x1 if the width changes]
             num_res_blocks x (x + block2(relu(block1(x))))                   block1 3x3, block2 1x1
             feature l = x
Activations are fp16 NHWC rows [B*h*w, C]; every convolution is one mos_gemm_bf16 launch (3x3 through the implicit-conv
path, the resnet add as its residual epilogue), the unshuffle, ReLU and pooling are mos_pixel_unshuffle / mos_relu_rows /
mos_avgpool2x (wrapped in adapter_ops.py).  No CPU / PyTorch fallback.
"""
import torch

from . import adapter_ops, ops

F16 = torch.float16
F32 = torch.float32


def adapter_param_shapes(in_channels, channels, num_res_blocks, downscale_factor=8):
    """{state-dict key: shape} of a full_adapter T2IAdapter"""
    s = {}

    def conv(name, co, ci, k):
        s[name + '.weight'] = (co, ci, k, k)
        s[name + '.bias'] = (co,)
    conv('adapter.conv_in', channels[0], in_channels * downscale_factor ** 2, 3)
    prev = channels[0]
    for l, c in enumerate(channels):
        if c != prev:
            conv(f'adapter.body.{l}.in_conv', c, prev, 1)
        for k in range(num_res_blocks):
            conv(f'adapter.body.{l}.resnets.{k}.block1', c, c, 3)
            conv(f'adapter.body.{l}.resnets.{k}.block2', c, c, 1)
        prev = c
    return s


def check_geometry(height, width, channels):
    """ValueError unless every level tiles: H, W multiples of 8 * 2^(L-1) (so AvgPool2d's ceil_mode never matters) and
    every width a multiple of the GEMM's 160-column tile"""
    down = 8 * 2 ** (len(channels) - 1)
    if height % down or width % down:
        raise ValueError(f'T2I-Adapter input {height} x {width}: height and width must be multiples of {down} '
                         f'(8 * 2^{len(channels) - 1} for {len(channels)} levels)')
    bad = [c for c in channels if c % 160]
    if bad:
        raise ValueError(f'T2I-Adapter channels {list(channels)}: every width must be a multiple of 160, {bad} are not')


class AdapterEngine:
    def __init__(self, state_dict, batch, height, width, in_channels=3, channels=(320, 640, 1280, 1280), num_res_blocks=2,
                 device='cuda'):
        """state_dict: diffusers-named tensors of T2IAdapter; height / width: condition-image size in pixels."""
        check_geometry(height, width, channels)
        self.dev = torch.device(device)
        self.B, self.H, self.W = batch, height, width
        self.cin, self.ch, self.nrb = in_channels, tuple(channels), num_res_blocks
        self.w, self.bufs = {}, {}
        self.launches = 0
        sd = state_dict
        self._pack(sd, 'adapter.conv_in', 3)
        prev = self.ch[0]
        for l, c in enumerate(self.ch):
            if c != prev:
                self._pack(sd, f'adapter.body.{l}.in_conv', 1)
            for k in range(self.nrb):
                self._pack(sd, f'adapter.body.{l}.resnets.{k}.block1', 3)
                self._pack(sd, f'adapter.body.{l}.resnets.{k}.block2', 1)
            prev = c

    def _pack(self, sd, name, k):
        """3x3: [Cout, Cin, 3, 3] -> tap-major [Cout, 9 Cin] fp16 (as VAEEngine._pack_conv3); 1x1: [Cout, Cin] fp16"""
        W = sd[name + '.weight'].detach().to(self.dev, F32)
        W = W.permute(0, 2, 3, 1).reshape(W.shape[0], -1) if k == 3 else W.reshape(W.shape[0], -1)
        self.w[name] = {'W': W.to(F16).contiguous(), 'bias': sd[name + '.bias'].detach().to(self.dev, F32).contiguous()}

    def buf(self, name, shape):
        key = (name, tuple(shape))
        if key not in self.bufs:
            self.bufs[key] = torch.empty(shape, device=self.dev, dtype=F16)
        return self.bufs[key]

    def gemm(self, A, name, out, *, M, conv=None, residual=None):
        ops.gemm(A, self.w[name]['W'], out, M=M, bias=self.w[name]['bias'], conv=conv, residual=residual)
        self.launches += 1
        return out

    @torch.no_grad()
    def forward(self, image):
        """image fp32 NCHW [B, Cin, H, W] (diffusers' preprocessing: [0, 1]) -> L fp16 NHWC row tensors [B*h_l*w_l, C_l]
        (h_0 = H / 8, halved per level).  The tensors are this engine's buffers: the next call overwrites them."""
        assert tuple(image.shape) == (self.B, self.cin, self.H, self.W), (tuple(image.shape), (self.B, self.cin, self.H, self.W))
        B = self.B
        h, w = self.H // 8, self.W // 8
        self.launches = 0
        K0 = 64 * self.cin
        x0 = self.buf('unshuffle', (B * h * w, K0))
        adapter_ops.pixel_unshuffle(image.to(self.dev, F32).contiguous(), x0)
        self.launches += 1
        x = self.gemm(x0, 'adapter.conv_in', self.buf('conv_in', (B * h * w, self.ch[0])), M=B * h * w,
                      conv=(B, h, w, K0))
        feats = []
        prev = self.ch[0]
        for l, c in enumerate(self.ch):
            if l > 0:
                p = self.buf(f'pool{l}', (B * (h // 2) * (w // 2), prev))
                adapter_ops.avgpool2x(x, p, B=B, H=h, W=w, C=prev)
                self.launches += 1
                h, w, x = h // 2, w // 2, p
            M = B * h * w
            if c != prev:
                x = self.gemm(x, f'adapter.body.{l}.in_conv', self.buf(f'in_conv{l}', (M, c)), M=M)
            for k in range(self.nrb):
                name = f'adapter.body.{l}.resnets.{k}'
                t = self.gemm(x, name + '.block1', self.buf(f't{l}', (M, c)), M=M, conv=(B, h, w, c))
                adapter_ops.relu_rows(t, M=M, C=c)
                self.launches += 1
                x = self.gemm(t, name + '.block2', self.buf(f'x{l}_{k % 2}', (M, c)), M=M, residual=x)
            feats.append(x)
            prev = c
        return feats
