"""UNetEngine — the SD1.5 UNet + ED-LoRA denoising step on the GPU, built only from libmos_sm100 kernels.

The engine owns the whole `unet(sample, t, encoder_hidden_states, cross_attention_kwargs,
down_block_additional_residuals).sample` call the reference makes at
mixofshow/pipelines/pipeline_edlora.py:277-282, trainer_edlora.py:237, gradient_fusion.py:619 and
pipeline_regionally_t2iadapter.py:556-566.  Activations are NHWC / token-major bf16; weights are packed once
(bf16, K-major, conv taps unrolled, q|k|v fused, GEGLU rows interleaved per 160-column tile, LoRA down padded to 16
rows and LoRA up pre-scaled by alpha).  Skip tensors are written by their producers straight into the channel slot
of the up-block concat buffer that will consume them, so `torch.cat([h, skip])` never moves a byte.

There is no CPU / PyTorch fallback: every arithmetic op below is a C-ABI call into the CUDA library.
"""
import math
import os

import torch

from . import ops
from ._lib import MOS_SEG_ROWS, MOS_SEG_TRANSPOSED

BF16 = torch.bfloat16       # weights (and the training engine's activations)
F16 = torch.float16
# split-K GEMMs are finalized by a separate mos_splitk_finalize launch; MOS_SPLITK_FUSED=1 (off by default) has the GEMM
# finalize in-kernel instead (mos_gemm_args.tile_counters), with the same summation order and bit-identical results
FUSED_SPLITK = os.environ.get('MOS_SPLITK_FUSED', '0') == '1'
# MOS_L2_PREFETCH=1 (off by default): every GEMM of the step stages the NEXT GEMM's weight matrix in L2 while it runs
# (mos_gemm_args.prefetch_ptr): the step streams 1.7 GB of weights through a mostly idle HBM, and the 50 MB L2 of an H100
# holds any single layer (at most 48 MB is staged).
L2_PREFETCH = os.environ.get('MOS_L2_PREFETCH', '0') == '1'
L2_PREFETCH_MAX_BYTES = 48 << 20
SPLITK_MIN_KB = int(os.environ.get('MOS_SPLITK_MIN_KB', '8'))      # fewest 64-deep k-blocks a split-K slice may get
SKIP_CH = [320, 320, 320, 320, 640, 640, 640, 1280, 1280, 1280, 1280, 1280]


def _r(x, m):
    return (x + m - 1) // m * m


def cross_attention_names(block_out=(320, 640, 1280, 1280), layers=2):
    """attn2 module names in reference order (edlora.py:176-190): down, mid, up; idx = position."""
    names = []
    nb = len(block_out)
    for i in range(nb - 1):
        for j in range(layers):
            names.append(f'down_blocks.{i}.attentions.{j}.transformer_blocks.0.attn2')
    names.append('mid_block.attentions.0.transformer_blocks.0.attn2')
    for i in range(1, nb):
        for j in range(layers + 1):
            names.append(f'up_blocks.{i}.attentions.{j}.transformer_blocks.0.attn2')
    return names


def level_sizes(height, width, levels):
    """latent (h, w) of every UNet level: diffusers' Downsample2D (3x3, stride 2, pad 1) gives ceil(h / 2) x ceil(w / 2),
    and each up block interpolates back to the size of the level above (forward_upsample_size), so the levels are exact
    halvings only when the latent sides are multiples of 2^(levels - 1)."""
    sizes = [(height, width)]
    for _ in range(levels - 1):
        h, w = sizes[-1]
        sizes.append(((h + 1) // 2, (w + 1) // 2))
    return sizes


def geglu_perm(n):
    """Row order of the packed GEGLU projection (n = 2H output rows): for every 160-column output tile, 80 rows of the value
    half followed by the matching 80 rows of the gate half, so that the fused epilogue finds both halves of an output
    column in one tile.  packed = natural[perm]."""
    half = n // 2
    assert half % 80 == 0
    return torch.cat([torch.cat([torch.arange(80 * t, 80 * t + 80), half + torch.arange(80 * t, 80 * t + 80)])
                      for t in range(half // 80)])


class UNetEngine:
    def __init__(self, state_dict, batch, height, width, *, lora=None, lora_alpha=1.0, merge_lora=False,
                 device='cuda', block_out=(320, 640, 1280, 1280), layers=2, heads=8, cross_dim=768, n_text=77,
                 emit_probs=False, use_graph=True, act_dtype=F16):
        """state_dict: diffusers-named fp32 tensors of the UNet.  lora: {f'{module}.lora_down.weight': [r,in],
        f'{module}.lora_up.weight': [out,r]} exactly as EDLoRATrainer.delta_state_dict()['unet'] stores it
        (trainer_edlora.py:371-378); rank <= 4.  batch includes the CFG duplication.  height/width: latent size.
        act_dtype: 16-bit type of every activation AND of the packed GEMM weights (wgmma takes one operand type for
        A and B).  Sampling uses fp16 - the reference's own sampling precision (README.md:146 torch_dtype=float16):
        with classifier-free guidance the scheduler consumes u + g (c - u), so the activation rounding noise of the two
        (nearly equal) halves is amplified by g; fp16's 3 extra mantissa bits bring the CFG-7.5 latents from 2.8e-3 (bf16,
        round 1) to < 5e-4 rel-L2 (tests/numerics_emulation.py).  Training keeps bf16 (gradient range)."""
        assert act_dtype in (F16, BF16)
        self.ACT = act_dtype
        self.dev = torch.device(device)
        self.B, self.H, self.W = batch, height, width
        self.block_out, self.layers, self.heads = tuple(block_out), layers, heads
        self.cross_dim, self.n_text = cross_dim, n_text
        self.emit_probs = emit_probs
        self.use_graph = use_graph
        self.lora = None if merge_lora else lora
        self.lora_alpha = float(lora_alpha)
        self._merge = lora if merge_lora else None
        self.sd = state_dict
        self.level_hw = level_sizes(height, width, len(block_out))
        self.w = {}
        self._pack_args = {}
        self.bufs = {}
        self.launches = 0
        self.xattn_names = cross_attention_names(block_out, layers)
        self._pack_all()
        self._alloc_io()
        self.graph = None
        self.regions = None     # list of (ehs_layers bf16 [16,B,77,768], (sh,sw,eh,ew) fractions)
        self.adapters = None    # list of 4 bf16 NHWC tensors [B*HW_l, C_l]
        self.region_hw = None   # (height, width) in pixels passed by the regional pipeline
        self.controller = None
        self.side = None        # side CUDA stream (created lazily on the device) for independent branches
        self.gram_rec = None    # gradient fusion: callable(key, A [M,C] bf16 view, M, C) fed with recorded GEMM inputs
        self._in_run, self._w_idx, self._w_seq, self._w_rec = False, 0, [], None      # L2 weight prefetch (see gemm())
        self.skip = set()       # profiling aid: op families not launched ('gemm','splitk','attn','gn','ln','misc')

    # ------------------------------------------------------------------------------------------ packing
    def _t(self, name):
        return self.sd[name].detach().to(self.dev, torch.float32)

    def _lora_pair(self, module):
        src = self._merge if self._merge is not None else self.lora
        if src is None:
            return None
        kd, ku = f'{module}.lora_down.weight', f'{module}.lora_up.weight'
        if kd not in src:
            return None
        d = src[kd].detach().to(self.dev, torch.float32)
        u = src[ku].detach().to(self.dev, torch.float32)
        return d.reshape(d.shape[0], -1), u.reshape(u.shape[0], -1)

    def _pack_linear(self, key, modules, geglu=False, conv3=False):
        """modules: list of module names whose weights are concatenated along N (q|k|v fusion)."""
        self._pack_args[key] = (list(modules), geglu, conv3)
        Ws, bs, downs, ups = [], [], [], []
        any_lora = False
        for m in modules:
            W = self._t(m + '.weight')
            if conv3:
                W = W.permute(0, 2, 3, 1).reshape(W.shape[0], -1)
            else:
                W = W.reshape(W.shape[0], -1)
            pair = self._lora_pair(m)
            if pair is not None and self._merge is not None:
                W = W + self.lora_alpha * (pair[1] @ pair[0])     # convert_edlora_to_diffusers.py:67-73
                pair = None
            Ws.append(W)
            bname = m + '.bias'
            bs.append(self._t(bname) if bname in self.sd else None)
            if pair is not None:
                any_lora = True
            downs.append(pair[0] if pair is not None else None)
            ups.append(pair[1] if pair is not None else None)
        W = torch.cat(Ws, 0)
        N, K = W.shape
        bias = None
        if any(b is not None for b in bs):
            bias = torch.cat([b if b is not None else torch.zeros(w_.shape[0], device=self.dev)
                              for b, w_ in zip(bs, Ws)])
        ent = {'N': N, 'K': K}
        perm = None
        if geglu:
            perm = geglu_perm(N).to(self.dev)
            W = W[perm]
            bias = bias[perm] if bias is not None else None
        ent['W'] = W.to(self.ACT).contiguous()
        ent['bias'] = bias.contiguous() if bias is not None else None
        if any_lora:
            assert len(modules) <= 4
            down16 = torch.zeros(16, K, device=self.dev)
            up = torch.zeros(N, 4, device=self.dev)
            off = 0
            for s, (d, u, w_) in enumerate(zip(downs, ups, Ws)):
                if d is not None:
                    r = d.shape[0]
                    assert r <= 4, 'LoRA rank > 4 is not supported by the fused epilogue'
                    down16[4 * s:4 * s + r] = d
                    up[off:off + w_.shape[0], :r] = u * self.lora_alpha
                off += w_.shape[0]
            if perm is not None:
                up = up[perm]
            ent['lora_down'] = down16.to(self.ACT).contiguous()
            ent['lora_up'] = up.contiguous()
            ent['lora_seg'] = Ws[0].shape[0] if len(modules) > 1 else N
        self.w[key] = ent
        return ent

    def _pack_norm(self, key, name):
        self.w[key] = (self._t(name + '.weight').contiguous(), self._t(name + '.bias').contiguous())

    def _resnet_names(self):
        names = []
        nb = len(self.block_out)
        for i in range(nb):
            for j in range(self.layers):
                names.append(f'down_blocks.{i}.resnets.{j}')
        names += ['mid_block.resnets.0', 'mid_block.resnets.1']
        for i in range(nb):
            for j in range(self.layers + 1):
                names.append(f'up_blocks.{i}.resnets.{j}')
        return names

    def _pack_all(self):
        sd = self.sd
        # time embedding + all time_emb_proj fused into one [sum Cout, 1280] GEMV
        self.w['t1'] = (self._t('time_embedding.linear_1.weight').to(BF16).contiguous(),
                        self._t('time_embedding.linear_1.bias').contiguous())
        self.w['t2'] = (self._t('time_embedding.linear_2.weight').to(BF16).contiguous(),
                        self._t('time_embedding.linear_2.bias').contiguous())
        ws, bs, self.temb_off = [], [], {}
        off = 0
        for rn in self._resnet_names():
            w_ = self._t(rn + '.time_emb_proj.weight')
            ws.append(w_)
            bs.append(self._t(rn + '.time_emb_proj.bias'))
            self.temb_off[rn] = off
            off += w_.shape[0]
        self.temb_total = off
        self.w['tproj'] = (torch.cat(ws, 0).to(BF16).contiguous(), torch.cat(bs, 0).contiguous())
        # conv_in / conv_out (fp32, CUDA-core edge kernels)
        ci = self._t('conv_in.weight')
        self.w['conv_in'] = (ci.permute(2, 3, 1, 0).reshape(-1, ci.shape[0]).contiguous(), self._t('conv_in.bias'))
        co = self._t('conv_out.weight')
        self.w['conv_out'] = (co.permute(0, 2, 3, 1).reshape(co.shape[0], 9, co.shape[1]).contiguous(),
                              self._t('conv_out.bias'))
        self._pack_norm('conv_norm_out', 'conv_norm_out')
        for rn in self._resnet_names():
            self._pack_norm(rn + '.norm1', rn + '.norm1')
            self._pack_norm(rn + '.norm2', rn + '.norm2')
            self._pack_linear(rn + '.conv1', [rn + '.conv1'], conv3=True)
            self._pack_linear(rn + '.conv2', [rn + '.conv2'], conv3=True)
            if rn + '.conv_shortcut.weight' in sd:
                self._pack_linear(rn + '.conv_shortcut', [rn + '.conv_shortcut'])
        for k in sd:
            if k.endswith('downsamplers.0.conv.weight') or k.endswith('upsamplers.0.conv.weight'):
                m = k[:-len('.weight')]
                self._pack_linear(m, [m], conv3=True)
        for an in self.xattn_names:
            tn = an[:-len('.transformer_blocks.0.attn2')]
            tb = tn + '.transformer_blocks.0'
            self._pack_norm(tn + '.norm', tn + '.norm')
            self._pack_linear(tn + '.proj_in', [tn + '.proj_in'])
            self._pack_linear(tn + '.proj_out', [tn + '.proj_out'])
            for n in ('norm1', 'norm2', 'norm3'):
                self._pack_norm(f'{tb}.{n}', f'{tb}.{n}')
            self._pack_linear(tb + '.attn1.qkv', [tb + '.attn1.to_q', tb + '.attn1.to_k', tb + '.attn1.to_v'])
            self._pack_linear(tb + '.attn1.out', [tb + '.attn1.to_out.0'])
            self._pack_linear(tb + '.attn2.q', [tb + '.attn2.to_q'])
            self._pack_linear(tb + '.attn2.kv', [tb + '.attn2.to_k', tb + '.attn2.to_v'])
            self._pack_linear(tb + '.attn2.out', [tb + '.attn2.to_out.0'])
            self._pack_linear(tb + '.ff1', [tb + '.ff.net.0.proj'], geglu=True)
            self._pack_linear(tb + '.ff2', [tb + '.ff.net.2'])
        self.sd = None  # drop the fp32 master copy reference

    # ------------------------------------------------------------------------------------------ buffers
    def buf(self, name, shape, dtype=None, zero=False):
        dtype = self.ACT if dtype is None else dtype
        key = (name, tuple(shape), dtype)
        if key not in self.bufs:
            self.bufs[key] = (torch.zeros if zero else torch.empty)(shape, device=self.dev, dtype=dtype)
        return self.bufs[key]

    def _alloc_io(self):
        B, H, W = self.B, self.H, self.W
        self.in_latents = torch.zeros(B, 4, H, W, device=self.dev)
        self.in_t = torch.zeros(B, device=self.dev)
        self.in_ehs = torch.zeros(len(self.xattn_names), B, self.n_text, self.cross_dim, device=self.dev, dtype=self.ACT)
        self.out_eps = torch.zeros(B, 4, H, W, device=self.dev)
        self.gn_partial = torch.zeros(B * 592 * 64, device=self.dev)   # GroupNorm fallback workspace: enough for any HW
        # concat buffers of the 12 up-block resnets: [h | skip]
        nb = len(self.block_out)
        rev = list(reversed(self.block_out))
        self.cat = []
        self.cat_ch = []
        skip_ch = [self.block_out[0]]
        for i, c in enumerate(self.block_out):
            skip_ch += [c] * self.layers
            if i < nb - 1:
                skip_ch.append(c)
        self.skip_ch = skip_ch
        h_ch = rev[0]
        k = 0
        for i in range(nb):
            lh, lw = self.level_hw[nb - 1 - i]
            M = B * lh * lw
            for j in range(self.layers + 1):
                cs = skip_ch[len(skip_ch) - 1 - k]
                ch = h_ch if j == 0 else rev[i]
                self.cat.append(torch.empty(M, ch + cs, device=self.dev, dtype=self.ACT))
                self.cat_ch.append((ch, cs))
                k += 1
            h_ch = rev[i]

    # ------------------------------------------------------------------------------------------ op helpers
    def _splits(self, M, N, kb_total):
        tiles = _r(M, 128) // 128 * (N // 160)
        if tiles >= 96 or kb_total < 2 * SPLITK_MIN_KB:
            return 1
        sms = torch.cuda.get_device_properties(self.dev).multi_processor_count   # the GEMM grid is one CTA per SM
        s = max(1, min(max(1, sms // tiles), kb_total // SPLITK_MIN_KB, 16))
        per = -(-kb_total // s)          # k blocks per split
        return -(-kb_total // per)       # normalised so that no split is empty

    def gemm(self, A, ent, out, *, M, conv=None, residual=None, bias_batch=None, rows_per_batch=0, geglu=False,
             heads=None, lda=None):
        K = ent['K'] // 9 if conv is not None else ent['K']
        kb_total = ent['K'] // 64
        lora = 'lora_down' in ent
        if 'gemm' in self.skip:
            return out
        splits = 1
        if not lora and not geglu and heads is None:
            splits = self._splits(M, ent['N'], kb_total)
        kw = dict(bias=ent['bias'], conv=conv, lda=lda)
        if L2_PREFETCH and self._in_run:
            # weight matrices in launch order: recorded on the first walk of the step, used by every later walk (the walk
            # is deterministic for a given engine state; a walk of a different length re-records)
            i = self._w_idx
            self._w_idx += 1
            if self._w_rec is not None:
                self._w_rec.append(ent['W'])
            elif i + 1 < len(self._w_seq) and self._w_seq[i] is ent['W']:
                nxt = self._w_seq[i + 1]
                if nxt.numel() * nxt.element_size() <= L2_PREFETCH_MAX_BYTES:
                    kw['prefetch'] = nxt
        if splits > 1:
            # the side stream (1x1 shortcuts, timestep MLP) runs concurrently with the main stream: its split-K launches
            # need a workspace and tile counters of their own
            on_side = self.side is not None and torch.cuda.current_stream() == self.side
            partial = (self.buf('splitk_side', (8 * 1024 * 1280,), torch.float32) if on_side
                       else self.buf('splitk', (16 * 1024 * 1280,), torch.float32))
            assert splits * M * ent['N'] <= partial.numel()
            if FUSED_SPLITK:
                # the `splits` CTAs of every output tile reduce the partials themselves (mos_gemm_args.tile_counters)
                ops.gemm(A, ent['W'], out, M=M, splits=splits, partial=partial, bias_batch=bias_batch, rows_per_batch=rows_per_batch, residual=residual,
                         bias_batch_ld=self.temb_total if bias_batch is not None else 0,
                         counters=self.buf('splitk_counters_side' if on_side else 'splitk_counters', (1024,), torch.int32,
                                           zero=True), **kw)
                self.launches += 1
                return out
            ops.gemm(A, ent['W'], None, M=M, splits=splits, partial=partial, conv=conv, lda=lda, prefetch=kw.get('prefetch'))
            if 'splitk' not in self.skip:
              ops.splitk_finalize(partial, splits, M, ent['N'], out, bias=ent['bias'], bias_batch=bias_batch,
                                  rows_per_batch=rows_per_batch, residual=residual,
                                  bias_batch_ld=self.temb_total if bias_batch is not None else 0)
            self.launches += 2
            return out
        if lora:
            kw.update(lora_down=ent['lora_down'], lora_up=ent['lora_up'], lora_seg=ent['lora_seg'])
        ops.gemm(A, ent['W'], out, M=M, residual=residual, bias_batch=bias_batch, rows_per_batch=rows_per_batch,
                 bias_batch_ld=self.temb_total if bias_batch is not None else 0, geglu=geglu, heads=heads,
                 **kw)
        self.launches += 1
        return out

    def groupnorm(self, x, key, y, *, HW, C, eps, silu):
        g, b = self.w[key]
        if 'gn' in self.skip:
            return
        ops.groupnorm(x, g, b, y, self.gn_partial, B=self.B, HW=HW, C=C, eps=eps, silu=silu, ldx=x.stride(0),
                      ldy=y.stride(0))
        self.launches += 1          # one-pass cluster kernel (two launches only on the large-slab fallback)

    def layernorm(self, x, key, y, *, M, C):
        g, b = self.w[key]
        if 'ln' in self.skip:
            return
        ops.layernorm(x, g, b, y, M=M, C=C, ldx=x.stride(0), ldy=y.stride(0))
        self.launches += 1

    def set_merged_lora(self, lora, lora_alpha=1.0, state_dict=None):
        """Gradient fusion runs the same UNet once per concept with that concept's LoRA folded into the weights
        (gradient_fusion.py:700-712): re-pack only the entries that contain a LoRA'd module instead of building a new
        engine (packing all 860 M parameters costs ~0.5 s)."""
        assert self.lora is None, 'set_merged_lora: the engine was built with an un-merged LoRA'
        if state_dict is None:
            raise ValueError('set_merged_lora needs the fp32 state_dict again (the engine keeps no master copy)')
        self.sd = state_dict
        old = self._merge or {}
        self._merge, self.lora_alpha = lora, float(lora_alpha)
        suffix = '.lora_down.weight'
        targets = {k[:-len(suffix)] for src in (old, lora or {}) for k in src if k.endswith(suffix)}
        for key, (modules, geglu, conv3) in list(self._pack_args.items()):
            if any(m in targets for m in modules):
                self._pack_linear(key, modules, geglu, conv3)
        self.sd = None
        self.graph = None
        self._text_version = None       # cached text K/V projections depend on the packed cross-attention weights

    # ------------------------------------------------------------------------------------------ blocks
    def resnet(self, name, x, out, h, w, cin, cout):
        """x: [M, cin] view (any row pitch); out: [M, cout] view.  ResnetBlock2D forward (SURVEY.md §9)."""
        B = self.B
        HW = h * w
        M = B * HW
        # the 1x1 shortcut only needs x: it runs on the side stream, concurrently with norm1 -> conv1 -> norm2
        res = x
        has_sc = name + '.conv_shortcut' in self.w
        if has_sc:
            main = torch.cuda.current_stream()
            self.side.wait_stream(main)
            with torch.cuda.stream(self.side):
                sc = self.buf('rn_sc', (M, cout))
                self.gemm(x, self.w[name + '.conv_shortcut'], sc, M=M, lda=x.stride(0))
            res = sc
        n1 = self.buf('rn_n', (M, cin))
        self.groupnorm(x, name + '.norm1', n1, HW=HW, C=cin, eps=1e-5, silu=True)
        h1 = self.buf('rn_h', (M, cout))
        tb = self.tproj[:, self.temb_off[name]:]
        self.gemm(n1, self.w[name + '.conv1'], h1, M=M, conv=(B, h, w, cin), bias_batch=tb, rows_per_batch=HW)
        n2 = self.buf('rn_n2', (M, cout))
        self.groupnorm(h1, name + '.norm2', n2, HW=HW, C=cout, eps=1e-5, silu=True)
        if has_sc:
            torch.cuda.current_stream().wait_stream(self.side)
        self.gemm(n2, self.w[name + '.conv2'], out, M=M, conv=(B, h, w, cout), residual=res)
        return out

    def _heads(self, segs, kinds, rows, C, tokens):
        d = C // self.heads
        return dict(seg_ptr=segs, seg_kind=kinds, seg_rows_pad=rows, heads=self.heads, head_dim=d,
                    dpad=_r(d, 64), dv_pad=_r(d, 16), tokens_per_batch=tokens)

    def _cross_kv(self, tb, ehs_layer, C, tag):
        B, T = self.B, self.n_text
        d = C // self.heads
        BH = B * self.heads
        Kc = self.buf(f'Kc{tag}', (BH, T, _r(d, 64)), zero=True)
        Vc = self.buf(f'Vc{tag}', (BH, _r(d, 16), _r(T, 8)), zero=True)
        A = ehs_layer.reshape(B * T, self.cross_dim)
        self.gemm(A, self.w[tb + '.attn2.kv'], None, M=B * T,
                  heads=self._heads([Kc, Vc], [MOS_SEG_ROWS, MOS_SEG_TRANSPOSED], [T, _r(T, 8)], C, T))
        return Kc, Vc

    def transformer(self, tn, x, out, h, w, C, xidx):
        """Transformer2DModel with one BasicTransformerBlock; x [M, C] view -> out [M, C] view."""
        B, Hh = self.B, self.heads
        N = h * w
        M = B * N
        d = C // Hh
        BH = B * Hh
        tb = tn + '.transformer_blocks.0'
        gn = self.buf('tr_gn', (M, C))
        self.groupnorm(x, tn + '.norm', gn, HW=N, C=C, eps=1e-6, silu=False)
        if self.gram_rec is not None:
            self.gram_rec(tn + '.proj_in', gn, M, C)
        t0 = self.buf('tr_t0', (M, C))
        self.gemm(gn, self.w[tn + '.proj_in'], t0, M=M)
        ln = self.buf('tr_ln', (M, C))
        # --- attn1 (self)
        self.layernorm(t0, tb + '.norm1', ln, M=M, C=C)
        if self.gram_rec is not None:
            self.gram_rec(tb + '.attn1.in', ln, M, C)
        Q = self.buf('Q', (BH, N, _r(d, 64)), zero=True)
        K = self.buf('K', (BH, N, _r(d, 64)), zero=True)
        Vt = self.buf('Vt', (BH, _r(d, 16), _r(N, 8)), zero=True)
        self.gemm(ln, self.w[tb + '.attn1.qkv'], None, M=M,
                  heads=self._heads([Q, K, Vt], [MOS_SEG_ROWS, MOS_SEG_ROWS, MOS_SEG_TRANSPOSED],
                                    [N, N, _r(N, 8)], C, N))
        ao = self.buf('tr_ao', (M, C))
        if 'attn' not in self.skip:
            ops.attention(Q, K, Vt, ao.view(B, N, C), batch=B, heads=Hh, head_dim=d, nq=N, nk=N)
        self.launches += 1
        if self.gram_rec is not None:
            self.gram_rec(tb + '.attn1.to_out.0', ao, M, C)
        t1 = self.buf('tr_t1', (M, C))
        self.gemm(ao, self.w[tb + '.attn1.out'], t1, M=M, residual=t0)
        # --- attn2 (cross, layer-wise text embedding: edlora.py:129-131)
        self.layernorm(t1, tb + '.norm2', ln, M=M, C=C)
        if self.gram_rec is not None:
            self.gram_rec(tb + '.attn2.to_q', ln, M, C)
        self.gemm(ln, self.w[tb + '.attn2.q'], None, M=M, heads=self._heads([Q], [MOS_SEG_ROWS], [N], C, N))
        if not self._kv_joined:     # the 16 text K/V projections were issued on the side stream at step start
            torch.cuda.current_stream().wait_stream(self.side)
            self._kv_joined = True
        Kc, Vc = self.kv[xidx]
        probs = None
        if self.emit_probs:
            probs = self.buf(f'probs{xidx}', (BH, N, self.n_text), torch.float32)
        if 'attn' not in self.skip:
            ops.attention(Q, Kc, Vc, ao.view(B, N, C), batch=B, heads=Hh, head_dim=d, nq=N, nk=self.n_text,
                          probs=probs)
        self.launches += 1
        if self.regions:
            self._region_rewrite(tb, Q, ao, h, w, C, xidx)
        if self.gram_rec is not None:
            self.gram_rec(tb + '.attn2.to_out.0', ao, M, C)
        t2 = self.buf('tr_t2', (M, C))
        self.gemm(ao, self.w[tb + '.attn2.out'], t2, M=M, residual=t1)
        # --- feed-forward (GEGLU fused in the first GEMM's epilogue)
        self.layernorm(t2, tb + '.norm3', ln, M=M, C=C)
        if self.gram_rec is not None:
            self.gram_rec(tb + '.ff.net.0.proj', ln, M, C)
        ff = self.buf('tr_ff', (M, 4 * C))
        self.gemm(ln, self.w[tb + '.ff1'], ff, M=M, geglu=True)
        if self.gram_rec is not None:
            self.gram_rec(tb + '.ff.net.2', ff, M, 4 * C)
        t3 = self.buf('tr_t3', (M, C))
        self.gemm(ff, self.w[tb + '.ff2'], t3, M=M, residual=t2)
        if self.gram_rec is not None:
            self.gram_rec(tn + '.proj_out', t3, M, C)
        self.gemm(t3, self.w[tn + '.proj_out'], out, M=M, residual=x)
        return out

    def _region_rewrite(self, tb, Q, ao, h, w, C, xidx):
        """RegionT2I_AttnProcessor.region_rewrite (pipeline_regionally_t2iadapter.py:32-86): per-region cross
        attention with the region's own K/V, mean over covering regions inside the boxes."""
        B, Hh = self.B, self.heads
        N = h * w
        d = C // Hh
        height, width = self.region_hw
        downscale = math.sqrt(height * width / N)                       # regional :45
        fh, fw = int(height // downscale), int(width // downscale)      # regional :48
        if (fh, fw) != (h, w):      # RegionallyT2IAdapterPipeline refuses these sizes up front (check_region_sizes)
            raise ValueError(f'region rule gives {fh} x {fw} for a {h} x {w} level at {height} x {width}')
        outs, boxes = [], []
        for r, (ehs_layers, box) in enumerate(self.regions):
            Kr, Vr = self.rkv[(r, xidx)]                  # step-invariant: projected once per prompt (update_text)
            o = self.buf(f'tr_ao_r{r}', (B * N, C))
            ops.attention(Q, Kr, Vr, o.view(B, N, C), batch=B, heads=Hh, head_dim=d, nq=N, nk=self.n_text)
            self.launches += 1
            sh, sw, eh, ew = box
            boxes.append((math.ceil(sh * fh), math.ceil(sw * fw), math.floor(eh * fh), math.floor(ew * fw)))
            outs.append(o)
        ptrs = self.buf(f'rptr_{N}', (len(outs),), torch.int64)
        if not torch.cuda.is_current_stream_capturing():
            ptrs.copy_(torch.tensor([o.data_ptr() for o in outs], dtype=torch.int64))
        ops.region_combine(ao, ptrs, boxes, ao, B=B, FH=fh, FW=fw, C=C, ld=C)
        self.launches += 1

    # ------------------------------------------------------------------------------------------ forward
    def _time(self):
        B = self.B
        emb = self.buf('temb0', (B, self.block_out[0]), torch.float32)
        ops.timestep_embedding(self.in_t, emb)
        t1 = self.buf('temb1', (B, 4 * self.block_out[0]), torch.float32)
        ops.gemv(emb, self.w['t1'][0], self.w['t1'][1], t1, act_out=True)
        t2 = self.buf('temb2', (B, 4 * self.block_out[0]), torch.float32)
        ops.gemv(t1, self.w['t2'][0], self.w['t2'][1], t2, act_out=True)       # stores SiLU(temb)
        self.tproj = self.buf('tproj', (B, self.temb_total), torch.float32)
        ops.gemv(t2, self.w['tproj'][0], self.w['tproj'][1], self.tproj)
        self.launches += 4

    def _skip_slot(self, i):
        k = len(self.cat) - 1 - i
        ch, cs = self.cat_ch[k]
        return self.cat[k][:, ch:ch + cs]

    def _xattn_channels(self):
        nb = len(self.block_out)
        ch = []
        for i in range(nb - 1):
            ch += [self.block_out[i]] * self.layers
        ch.append(self.block_out[-1])
        rev = list(reversed(self.block_out))
        for i in range(1, nb):
            ch += [rev[i]] * (self.layers + 1)
        return ch

    def update_text(self):
        """Text K / V projections (+ LoRA) of the 16 cross-attention layers, and of every region's embeddings: they depend on
        the prompt only, not on the denoise step (the reference recomputes them every step, edlora.py:143-145,
        pipeline_regionally_t2iadapter.py:120-129), so they are projected ONCE per prompt, outside the captured step.
        `run()` calls this whenever `in_ehs` / the region embeddings have been written since (tensor version counters)."""
        launches = self.launches
        self.kv, self.rkv = {}, {}
        for xidx, (an, C) in enumerate(zip(self.xattn_names, self._xattn_channels())):
            tbn = an[:-len('.attn2')]
            self.kv[xidx] = self._cross_kv(tbn, self.in_ehs[xidx], C, f'_x{xidx}')
            for r, (ehs_layers, _) in enumerate(self.regions or []):
                self.rkv[(r, xidx)] = self._cross_kv(tbn, ehs_layers[xidx], C, f'_r{r}_{xidx}')
        self.text_launches = self.launches - launches
        self.launches = launches
        self._text_version = self._text_state()

    def _text_state(self):
        return (self.in_ehs._version,) + tuple(e._version for e, _ in (self.regions or []))

    def _run(self):
        B, H, W = self.B, self.H, self.W
        nb = len(self.block_out)
        if getattr(self, '_text_version', None) != self._text_state() and not torch.cuda.is_current_stream_capturing():
            self.update_text()
        self.launches = 0
        self._in_run, self._w_idx = True, 0
        self._w_rec = [] if (L2_PREFETCH and not self._w_seq) else None
        # side stream: timestep MLP + all 22 time_emb_proj, concurrently with conv_in on the main stream
        main = torch.cuda.current_stream()
        if self.side is None:
            self.side = torch.cuda.Stream(device=self.dev)
            self.ev_time = torch.cuda.Event()
        self.side.wait_stream(main)
        with torch.cuda.stream(self.side):
            self._time()
            self.ev_time.record(self.side)
        self._kv_joined = True
        si = 0
        x = self._skip_slot(si)
        ops.conv_in(self.in_latents, self.w['conv_in'][0], self.w['conv_in'][1], x, ldy=x.stride(0))
        self.launches += 1
        si += 1
        main.wait_event(self.ev_time)      # resnets need the time_emb_proj table
        h, w, cin = H, W, self.block_out[0]
        xi = 0
        for i, c in enumerate(self.block_out):
            has_attn = i < nb - 1
            for j in range(self.layers):
                slot = self._skip_slot(si)
                si += 1
                M = B * h * w
                if has_attn:
                    r = self.buf('blk_r', (M, c))
                    self.resnet(f'down_blocks.{i}.resnets.{j}', x, r, h, w, cin, c)
                    self.transformer(f'down_blocks.{i}.attentions.{j}', r, slot, h, w, c, xi)
                    xi += 1
                else:
                    self.resnet(f'down_blocks.{i}.resnets.{j}', x, slot, h, w, cin, c)
                x, cin = slot, c
                if j == self.layers - 1 and self.adapters is not None:
                    a = self.adapters[i]
                    ops.add_rows(x, a, M=M, C=c, ldx=x.stride(0), ldr=a.stride(0))
                    self.launches += 1
            if has_attn:
                slot = self._skip_slot(si)
                si += 1
                ho, wo = self.level_hw[i + 1]
                Mo = B * ho * wo
                col = self.buf('im2col', (Mo, 9 * c))
                ops.im2col_s2(x, col, B=B, H=h, W=w, C=c, ldx=x.stride(0))
                self.launches += 1
                self.gemm(col, self.w[f'down_blocks.{i}.downsamplers.0.conv'], slot, M=Mo)
                h, w = ho, wo
                x = slot
        # mid
        c = self.block_out[-1]
        M = B * h * w
        r = self.buf('blk_r', (M, c))
        self.resnet('mid_block.resnets.0', x, r, h, w, c, c)
        r2 = self.buf('blk_r2', (M, c))
        self.transformer('mid_block.attentions.0', r, r2, h, w, c, xi)
        xi += 1
        k = 0
        dst = self.cat[0][:, :self.cat_ch[0][0]]
        self.resnet('mid_block.resnets.1', r2, dst, h, w, c, c)
        # up
        rev = list(reversed(self.block_out))
        for i, c in enumerate(rev):
            has_attn = i > 0
            for j in range(self.layers + 1):
                M = B * h * w
                ch, cs = self.cat_ch[k]
                xin = self.cat[k]
                last_in_block = j == self.layers
                final = last_in_block and i == nb - 1
                if final:
                    nxt = self.buf('final', (M, c))
                elif last_in_block:
                    nxt = self.buf('up_pre', (M, c))
                else:
                    nxt = self.cat[k + 1][:, :self.cat_ch[k + 1][0]]
                if has_attn:
                    r = self.buf('blk_r', (M, c))
                    self.resnet(f'up_blocks.{i}.resnets.{j}', xin, r, h, w, ch + cs, c)
                    self.transformer(f'up_blocks.{i}.attentions.{j}', r, nxt, h, w, c, xi)
                    xi += 1
                else:
                    self.resnet(f'up_blocks.{i}.resnets.{j}', xin, nxt, h, w, ch + cs, c)
                k += 1
                if last_in_block and not final:
                    # diffusers' forward_upsample_size: up to the size of the skip this level concatenates
                    ho, wo = self.level_hw[nb - 2 - i]
                    up = self.buf('up_x', (B * ho * wo, c))
                    ops.upsample2x(nxt, up, B=B, H=h, W=w, C=c, ldx=nxt.stride(0), Ho=ho, Wo=wo)
                    self.launches += 1
                    h, w = ho, wo
                    dst = self.cat[k][:, :self.cat_ch[k][0]]
                    self.gemm(up, self.w[f'up_blocks.{i}.upsamplers.0.conv'], dst, M=B * h * w, conv=(B, h, w, c))
        # out
        M = B * h * w
        fin = self.buf('final', (M, self.block_out[0]))
        fn = self.buf('final_n', (M, self.block_out[0]))
        self.groupnorm(fin, 'conv_norm_out', fn, HW=h * w, C=self.block_out[0], eps=1e-5, silu=True)
        ops.conv_out(fn, self.w['conv_out'][0], self.w['conv_out'][1], self.out_eps, B=B, H=h, W=w,
                     C=self.block_out[0])
        self.launches += 1
        self._in_run = False
        if self._w_rec is not None:
            self._w_seq, self._w_rec = self._w_rec, None
        elif L2_PREFETCH and self._w_idx != len(self._w_seq):
            self._w_seq = []                 # the walk changed (regions / adapters switched): re-record on the next walk

    def set_regions(self, regions, region_hw):
        """regions: list of (ehs_layers bf16 [n_layers,B,77,768], (sh,sw,eh,ew) box fractions) or None.  The embeddings
        are copied into static buffers; the captured graph is invalidated only when the box signature changes."""
        sig = None if not regions else (tuple(tuple(float(v) for v in b) for _, b in regions), tuple(region_hw))
        if sig != getattr(self, '_region_sig', None):
            self.graph = None
            self._region_sig = sig
        if not regions:
            self.regions, self.region_hw = None, None
            return
        static = []
        for r, (emb, box) in enumerate(regions):
            buf = self.buf(f'region_ehs{r}', tuple(self.in_ehs.shape))
            buf.copy_(emb)
            static.append((buf, tuple(float(v) for v in box)))
        self.regions, self.region_hw = static, tuple(region_hw)

    def set_adapters(self, adapters):
        """adapters: list of per-down-block residuals as NHWC bf16 [B*HW_l, C_l] (T2I-Adapter features) or None."""
        has = adapters is not None
        if has != (self.adapters is not None):
            self.graph = None
        if not has:
            self.adapters = None
            return
        static = []
        for l, a in enumerate(adapters):
            buf = self.buf(f'adapter{l}', tuple(a.shape))
            buf.copy_(a)
            static.append(buf)
        self.adapters = static

    def forward(self, latents, timesteps, ehs_layers):
        """latents fp32 NCHW [B,4,H,W]; timesteps [B]; ehs_layers [16,B,77,768] (layer-major). -> eps fp32 NCHW."""
        self.in_latents.copy_(latents)
        self.in_t.copy_(timesteps.to(self.dev, torch.float32).expand(self.B))
        self.in_ehs.copy_(ehs_layers)
        self.run()
        return self.out_eps

    def run(self):
        if getattr(self, '_text_version', None) != self._text_state():
            self.update_text()
        if not self.use_graph or self.emit_probs:
            self._run()
            return
        if self.graph is None:
            # warm-up (allocates every scratch buffer, sets kernel attributes) then capture
            s = torch.cuda.Stream()
            s.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(s):
                self._run()
                if L2_PREFETCH and not self._w_seq:
                    self._run()              # the walk changed since the weight order was recorded: record it again
            torch.cuda.current_stream().wait_stream(s)
            torch.cuda.synchronize()
            self.graph = torch.cuda.CUDAGraph()
            with torch.cuda.graph(self.graph):
                self._run()
        self.graph.replay()


def ehs_to_layer_major(ehs, n_layers=16, dtype=F16):
    """[B,16,77,768] (pipeline layout, pipeline_edlora.py:145) or [B,77,768] -> 16-bit [16,B,77,768] (the engine's
    activation type; `in_ehs.copy_()` converts if they differ)."""
    if ehs.ndim == 3:
        ehs = ehs[:, None].expand(-1, n_layers, -1, -1)
    elif ehs.shape[1] > n_layers:      # a smaller topology uses the first n_layers embeddings (idx < n_layers)
        ehs = ehs[:, :n_layers]
    assert ehs.shape[1] == n_layers, f'need {n_layers} layer-wise embeddings, got {ehs.shape[1]}'
    return ehs.permute(1, 0, 2, 3).to(dtype).contiguous()
