"""VAEEngine — the SD1.5 `AutoencoderKL` encoder and decoder on the GPU (SURVEY.md 8f rank 2), built only from libmos_sm100
kernels.  Owns the two calls the reference makes:

    latents = self.vae.encode(images).latent_dist.sample() * 0.18215     mixofshow/pipelines/trainer_edlora.py:203-204
    image   = self.vae.decode(latents / 0.18215).sample                   mixofshow/pipelines/pipeline_edlora.py:303-313

diffusers-0.19.3 topology (block_out (128, 256, 512, 512), 2 layers per encoder block / 3 per decoder block, GroupNorm(32,
eps 1e-6) + SiLU + 3x3 conv resnets without time embedding, one single-head attention of width 512 in each mid block,
asymmetric-padded stride-2 downsampling, nearest x2 upsampling).  Activations are fp16 NHWC, weights fp16 (inference).

Shapes are bent to the GEMM kernel's 160-column tiles without touching the arithmetic: a C-channel tensor lives in a
[M, Cp] buffer (Cp = C rounded up to 160: 128 -> 160, 256 -> 320, 512 -> 640) whose pad columns are written as zeros (zero
weight rows, zero bias); reductions run over the C real channels (pixel pitch Cp).  The d = 512 attention is
S = Q K^T (wgmma GEMM, fp32 out) -> mos_softmax_rows -> O = P V (wgmma GEMM): the 4096 x 4096 logits of a 512^2 image
are 68 MB, once per image.  No CPU / PyTorch fallback: every arithmetic op is a C-ABI call.
"""
import torch

from . import ops
from ._lib import MOS_SEG_ROWS, MOS_SEG_TRANSPOSED

F16 = torch.float16
F32 = torch.float32


def _r(x, m):
    return (x + m - 1) // m * m


class VAEEngine:
    def __init__(self, state_dict, batch, height, width, *, device='cuda', block_out=(128, 256, 512, 512), layers=2,
                 latent_channels=4, scaling_factor=0.18215, encoder=True, decoder=True):
        """state_dict: diffusers-named fp32 tensors of AutoencoderKL.  height / width: IMAGE size in pixels (multiples of
        2^(len(block_out) - 1) * 8 so that every level tiles)."""
        self.dev = torch.device(device)
        self.B, self.H, self.W = batch, height, width
        self.ch, self.L, self.lat = tuple(block_out), layers, latent_channels
        self.scaling = float(scaling_factor)
        self.down = 2 ** (len(self.ch) - 1)
        assert height % self.down == 0 and width % self.down == 0
        self.sd = state_dict
        self.w, self.bufs = {}, {}
        self.launches = 0
        self.has_enc, self.has_dec = encoder, decoder
        if encoder:
            self._pack_encoder()
        if decoder:
            self._pack_decoder()
        self.sd = None

    # ------------------------------------------------------------------------------------------ packing
    def _t(self, name):
        return self.sd[name].detach().to(self.dev, F32)

    def _pack_conv3(self, key, name, cout_pad=None):
        """3x3 conv weights [Cout, Cin, 3, 3] -> tap-major [Np, 9 * Cin] fp16 (Np = Cout rounded up to 160, zero rows)."""
        W = self._t(name + '.weight')
        co, ci = W.shape[0], W.shape[1]
        Np = _r(co, 160) if cout_pad is None else cout_pad
        Wp = torch.zeros(Np, 9 * ci, device=self.dev)
        Wp[:co] = W.permute(0, 2, 3, 1).reshape(co, -1)
        b = torch.zeros(Np, device=self.dev)
        b[:co] = self._t(name + '.bias')
        self.w[key] = {'W': Wp.to(F16).contiguous(), 'bias': b.contiguous(), 'N': Np, 'cin': ci, 'cout': co}

    def _pack_lin(self, key, names, pad_each=None):
        """1x1 conv / Linear weights of `names` concatenated along N, each padded to `pad_each` rows; K padded with zero
        columns to a multiple of 64 is not needed (all widths are multiples of 64)."""
        Ws, bs = [], []
        for n in names:
            W = self._t(n + '.weight')
            W = W.reshape(W.shape[0], -1)
            co = W.shape[0]
            Np = _r(co, 160) if pad_each is None else pad_each
            Wp = torch.zeros(Np, W.shape[1], device=self.dev)
            Wp[:co] = W
            b = torch.zeros(Np, device=self.dev)
            if n + '.bias' in self.sd:
                b[:co] = self._t(n + '.bias')
            Ws.append(Wp)
            bs.append(b)
        self.w[key] = {'W': torch.cat(Ws, 0).to(F16).contiguous(), 'bias': torch.cat(bs, 0).contiguous()}

    def _pack_norm(self, key, name):
        self.w[key] = (self._t(name + '.weight').contiguous(), self._t(name + '.bias').contiguous())

    def _pack_resnet(self, name):
        self._pack_norm(name + '.norm1', name + '.norm1')
        self._pack_norm(name + '.norm2', name + '.norm2')
        self._pack_conv3(name + '.conv1', name + '.conv1')
        self._pack_conv3(name + '.conv2', name + '.conv2')
        if name + '.conv_shortcut.weight' in self.sd:
            self._pack_lin(name + '.conv_shortcut', [name + '.conv_shortcut'])

    def _pack_mid(self, pre):
        for j in (0, 1):
            self._pack_resnet(f'{pre}.mid_block.resnets.{j}')
        a = f'{pre}.mid_block.attentions.0'
        self._pack_norm(a + '.group_norm', a + '.group_norm')
        C = self.ch[-1]
        Cp = _r(C, 160)
        # q | k | v as three "heads" segments of width Cp (one head of dim Cp, pad rows zero): the head-split epilogue
        # writes Q, K as contiguous [B, tokens, Cp] rows and V^T as [B, Cp, tokens]
        self._pack_lin(a + '.qkv', [a + '.to_q', a + '.to_k', a + '.to_v'], pad_each=Cp)
        # out projection reads the Cp-wide attention output (zero pad columns): K padded with zero columns
        W = self._t(a + '.to_out.0.weight')
        Wp = torch.zeros(Cp, Cp, device=self.dev)
        Wp[:C, :C] = W
        b = torch.zeros(Cp, device=self.dev)
        b[:C] = self._t(a + '.to_out.0.bias')
        self.w[a + '.out'] = {'W': Wp.to(F16).contiguous(), 'bias': b.contiguous()}

    def _pack_encoder(self):
        ci = self._t('encoder.conv_in.weight')
        self.w['enc.conv_in'] = (ci.permute(2, 3, 1, 0).reshape(-1, ci.shape[0]).contiguous(), self._t('encoder.conv_in.bias'))
        for i in range(len(self.ch)):
            for j in range(self.L):
                self._pack_resnet(f'encoder.down_blocks.{i}.resnets.{j}')
            if i < len(self.ch) - 1:
                n = f'encoder.down_blocks.{i}.downsamplers.0.conv'
                self._pack_conv3(n, n)
        self._pack_mid('encoder')
        self._pack_norm('encoder.conv_norm_out', 'encoder.conv_norm_out')
        self._pack_conv3('encoder.conv_out', 'encoder.conv_out')
        self.w['quant'] = (self._t('quant_conv.weight').reshape(2 * self.lat, 2 * self.lat).contiguous(),
                           self._t('quant_conv.bias').contiguous())

    def _pack_decoder(self):
        self.w['post_quant'] = (self._t('post_quant_conv.weight').reshape(self.lat, self.lat).contiguous(),
                                self._t('post_quant_conv.bias').contiguous())
        ci = self._t('decoder.conv_in.weight')
        self.w['dec.conv_in'] = (ci.permute(2, 3, 1, 0).reshape(-1, ci.shape[0]).contiguous(), self._t('decoder.conv_in.bias'))
        self._pack_mid('decoder')
        for i in range(len(self.ch)):
            for j in range(self.L + 1):
                self._pack_resnet(f'decoder.up_blocks.{i}.resnets.{j}')
            if i < len(self.ch) - 1:
                n = f'decoder.up_blocks.{i}.upsamplers.0.conv'
                self._pack_conv3(n, n)
        self._pack_norm('decoder.conv_norm_out', 'decoder.conv_norm_out')
        co = self._t('decoder.conv_out.weight')
        self.w['dec.conv_out'] = (co.permute(0, 2, 3, 1).reshape(co.shape[0], 9, co.shape[1]).contiguous(),
                                  self._t('decoder.conv_out.bias'))

    # ------------------------------------------------------------------------------------------ op helpers
    def buf(self, name, shape, dtype=F16, zero=False):
        key = (name, tuple(shape), dtype)
        if key not in self.bufs:
            self.bufs[key] = (torch.zeros if zero else torch.empty)(shape, device=self.dev, dtype=dtype)
        return self.bufs[key]

    def gemm(self, A, ent, out, *, M, conv=None, residual=None, lda=None, heads=None, out_f32=False):
        ops.gemm(A, ent['W'], out, M=M, bias=ent.get('bias'), conv=conv, residual=residual, lda=lda, heads=heads,
                 out_f32=out_f32)
        self.launches += 1
        return out

    def groupnorm(self, x, key, y, *, HW, C, silu):
        g, b = self.w[key]
        part = self.buf('gn_partial', (self.B * 592 * 64,), F32, zero=True)
        ops.groupnorm(x, g, b, y, part, B=self.B, HW=HW, C=C, eps=1e-6, silu=silu, ldx=x.stride(0), ldy=y.stride(0))
        self.launches += 1

    def resnet(self, name, x, h, w, cin, cout, tag):
        """x: [M, Cp(cin)] -> new [M, Cp(cout)] buffer (ResnetBlock2D without time embedding, oracle/vae.py)."""
        B = self.B
        HW = h * w
        M = B * HW
        n1 = self.buf('n_a', (M, cin))
        self.groupnorm(x, name + '.norm1', n1, HW=HW, C=cin, silu=True)
        h1 = self.buf('h_a', (M, _r(cout, 160)))
        self.gemm(n1, self.w[name + '.conv1'], h1, M=M, conv=(B, h, w, cin))
        n2 = self.buf('n_b', (M, cout))
        self.groupnorm(h1, name + '.norm2', n2, HW=HW, C=cout, silu=True)
        res = x
        if name + '.conv_shortcut' in self.w:
            res = self.buf('sc', (M, _r(cout, 160)))
            self.gemm(x, self.w[name + '.conv_shortcut'], res, M=M, lda=x.stride(0))
        out = self.buf(f'x_{tag}', (M, _r(cout, 160)))
        self.gemm(n2, self.w[name + '.conv2'], out, M=M, conv=(B, h, w, cout), residual=res)
        return out

    def attention(self, a, x, h, w, C):
        """Single-head attention block with GroupNorm and residual (oracle/vae.py Attention); x [M, Cp] -> new buffer."""
        B = self.B
        N = h * w
        M = B * N
        Cp = _r(C, 160)
        gn = self.buf('at_gn', (M, C))
        self.groupnorm(x, a + '.group_norm', gn, HW=N, C=C, silu=False)
        Nk = _r(N, 160)                                       # keys padded to the GEMM tile (zero rows, masked by softmax)
        Np = _r(N, 64)               # the P V GEMM's depth: P's columns and V's tokens past N stay zero (odd latent sizes)
        Q = self.buf('at_Q', (B, N, Cp), zero=True)
        K = self.buf('at_K', (B, Nk, Cp), zero=True)
        Vt = self.buf('at_Vt', (B, Cp, Np), zero=True)
        hseg = dict(seg_ptr=[Q, K, Vt], seg_kind=[MOS_SEG_ROWS, MOS_SEG_ROWS, MOS_SEG_TRANSPOSED], seg_rows_pad=[N, Nk, Np],
                    heads=1, head_dim=Cp, dpad=Cp, dv_pad=Cp, tokens_per_batch=N)
        self.gemm(gn, self.w[a + '.qkv'], None, M=M, heads=hseg)
        S = self.buf('at_S', (N, Nk), F32)
        P = self.buf('at_P', (N, Np), zero=True)
        O = self.buf('at_O', (M, Cp))
        for b in range(B):
            ops.gemm(Q[b], K[b], S, M=N, out_f32=True)                           # S = Q K^T   [N, Nk] fp32
            ops.softmax_rows(S, P, rows=N, cols=N, scale=C ** -0.5)
            ops.gemm(P, Vt[b], O[b * N:(b + 1) * N], M=N)                        # O = P V     [N, Cp]
            self.launches += 3
        out = self.buf('x_at', (M, Cp))
        self.gemm(O, self.w[a + '.out'], out, M=M, residual=x)
        return out

    def mid(self, pre, x, h, w):
        C = self.ch[-1]
        x = self.resnet(f'{pre}.mid_block.resnets.0', x, h, w, C, C, 'm0')
        x = self.attention(f'{pre}.mid_block.attentions.0', x, h, w, C)
        return self.resnet(f'{pre}.mid_block.resnets.1', x, h, w, C, C, 'm1')

    # ------------------------------------------------------------------------------------------ encode / decode
    @torch.no_grad()
    def encode(self, images, noise=None):
        """images fp32 NCHW [B, 3, H, W] in [-1, 1] -> (mean, logvar) fp32 [B, 4, H/8, W/8]; with `noise` (standard normal,
        same shape as the mean) also the scaled latent sample `0.18215 * (mean + std * noise)` (trainer_edlora.py:203-204)."""
        assert self.has_enc and tuple(images.shape) == (self.B, 3, self.H, self.W)
        B, h, w = self.B, self.H, self.W
        self.launches = 0
        c0 = self.ch[0]
        x = self.buf('x_in', (B * h * w, _r(c0, 160)), zero=True)
        ops.conv_in(images.to(self.dev, F32).contiguous(), self.w['enc.conv_in'][0], self.w['enc.conv_in'][1], x,
                    ldy=x.stride(0))
        cin = c0
        for i, c in enumerate(self.ch):
            for j in range(self.L):
                x = self.resnet(f'encoder.down_blocks.{i}.resnets.{j}', x, h, w, cin, c, f'e{(i * self.L + j) & 1}')
                cin = c
            if i < len(self.ch) - 1:
                Mo = B * (h // 2) * (w // 2)
                col = self.buf('im2col', (Mo, 9 * c))
                ops.im2col_s2(x, col, B=B, H=h, W=w, C=c, ldx=x.stride(0), pad=0)
                h, w = h // 2, w // 2
                nx = self.buf(f'x_d{i}', (Mo, _r(c, 160)))
                self.gemm(col, self.w[f'encoder.down_blocks.{i}.downsamplers.0.conv'], nx, M=Mo)
                x = nx
                self.launches += 1
        x = self.mid('encoder', x, h, w)
        C = self.ch[-1]
        M = B * h * w
        n = self.buf('n_a', (M, C))
        self.groupnorm(x, 'encoder.conv_norm_out', n, HW=h * w, C=C, silu=True)
        mo = self.buf('moments', (M, 160))
        self.gemm(n, self.w['encoder.conv_out'], mo, M=M, conv=(B, h, w, C))
        mean = torch.empty(B, self.lat, h, w, device=self.dev)
        logvar = torch.empty_like(mean)
        latents = None
        if noise is not None:
            noise = noise.to(self.dev, F32).contiguous()
            latents = torch.empty_like(mean)
        ops.vae_moments(mo, self.w['quant'][0], self.w['quant'][1], mean, logvar, B=B, HW=h * w, L=self.lat, noise=noise,
                        scaling=self.scaling, latents=latents)
        self.launches += 2
        return (mean, logvar) if noise is None else (mean, logvar, latents)

    @torch.no_grad()
    def decode(self, z):
        """z fp32 NCHW [B, 4, H/8, W/8] (UN-scaled: the caller divides by 0.18215, pipeline_edlora.py:304) -> image fp32
        NCHW [B, 3, H, W]."""
        assert self.has_dec
        B = self.B
        h, w = self.H // self.down, self.W // self.down
        assert tuple(z.shape) == (B, self.lat, h, w)
        self.launches = 0
        zq = torch.empty(B, self.lat, h, w, device=self.dev)
        ops.conv1x1_nchw(z.to(self.dev, F32).contiguous(), self.w['post_quant'][0], self.w['post_quant'][1], zq)
        C = self.ch[-1]
        x = self.buf('x_zin', (B * h * w, _r(C, 160)), zero=True)
        ops.conv_in(zq, self.w['dec.conv_in'][0], self.w['dec.conv_in'][1], x, ldy=x.stride(0))
        x = self.mid('decoder', x, h, w)
        rev = list(reversed(self.ch))
        cin = rev[0]
        for i, c in enumerate(rev):
            for j in range(self.L + 1):
                x = self.resnet(f'decoder.up_blocks.{i}.resnets.{j}', x, h, w, cin, c, f'u{(i * 3 + j) & 1}')
                cin = c
            if i < len(rev) - 1:
                up = self.buf('up', (B * 4 * h * w, c))
                ops.upsample2x(x, up, B=B, H=h, W=w, C=c, ldx=x.stride(0))
                h, w = 2 * h, 2 * w
                nx = self.buf(f'x_up{i}', (B * h * w, _r(c, 160)))
                self.gemm(up, self.w[f'decoder.up_blocks.{i}.upsamplers.0.conv'], nx, M=B * h * w, conv=(B, h, w, c))
                x = nx
                self.launches += 1
        c0 = self.ch[0]
        n = self.buf('n_out', (B * h * w, c0))
        self.groupnorm(x, 'decoder.conv_norm_out', n, HW=h * w, C=c0, silu=True)
        img = torch.empty(B, 3, h, w, device=self.dev)
        ops.conv_out(n, self.w['dec.conv_out'][0], self.w['dec.conv_out'][1], img, B=B, H=h, W=w, C=c0)
        self.launches += 3
        return img
