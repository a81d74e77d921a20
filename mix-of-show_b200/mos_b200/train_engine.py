"""TrainEngine — the UNet side of one ED-LoRA training step on the GPU (EDLoRATrainer.forward from `add_noise` to the
loss, trainer_edlora.py:218-261, the `loss.backward()` of train_edlora.py:120-123 and the AdamW update of the UNet LoRA
group, train_edlora.py:57,129), built only from libmos_sm100 kernels.

All base weights are frozen (trainer_edlora.py:88-90): the backward pass produces activation gradients (tensor-core
GEMMs on transposed weight packs, flash-attention backward, GroupNorm / LayerNorm / GEGLU backward) and the rank-4 LoRA
gradients, accumulated into ONE flat fp32 buffer (dp.FlatTrainState) so that the data-parallel step needs a single
all-reduce (SURVEY.md §8e).  The LoRA placement is the reference's `where` (trainer_edlora.py:121-133): `Attention` = the
128 attention projections; `Transformer2DModel` adds proj_in, proj_out (1x1 convs), ff.net.0.proj (GEGLU) and ff.net.2 of
every transformer block.  The GEGLU projection's LoRA up lives in the flat state in the packed row order of its GEMM
(engine.geglu_perm; AdamW is elementwise); `load_lora_state_dict` / `lora_state_dict` / `lora_grad_dict` speak the module's
natural order.  The attention regulariser (cal_attn_reg, :263-313) only
ever reads two key columns of the cross-attention maps, so the forward emits exactly those columns.

With `lora=None` the UNet is frozen (only text-side groups train): the forward runs plain GEMM epilogues and the backward
runs the full dX chain down to d(text embeddings) with no LoRA-gradient or LoRA-pack launch and no LoRA rows in the
backward packs.  The text encoder is attached with `attach_text_engine`: a training CLIPTrainEngine (text_grad=True) or a
frozen CLIPTextEngine whose forward runs inside the same captured step (text_grad=False: no d(text embeddings) and no text
K / V dX GEMMs).

With `shared_ehs=True` (vanilla LoRA, the reference's `enable_edlora: false`, trainer_edlora.py:220-234) every
cross-attention layer reads ONE text embedding: `in_ehs` is [1, B, 77, 768] instead of the layer-major [16, B, 77, 768],
the text encoder runs over B sequences, and d(text embedding) is the sum over the 16 layers of dK_l (W_k + a U_k D_k) +
dV_l (W_v + a U_v D_v), accumulated in fp32 by the GEMM's fp32 output path (`accumulate`) in the backward's fixed layer
order (so the step stays bit-reproducible) and rounded to bf16 once for the text encoder's backward.
"""
import math

import torch

from . import ops
from ._lib import MOS_SEG_ROWS
from .dp import FlatTrainState
from .engine import BF16, UNetEngine, _r, geglu_perm

F32 = torch.float32
_PROJ = ('to_q', 'to_k', 'to_v', 'to_out.0')
UNET_WHERE = ('Attention', 'Transformer2DModel')
_GEGLU = '.ff.net.0.proj'


def _key(t):
    return (t.data_ptr(), t.shape[0], t.shape[1])


class TrainEngine(UNetEngine):
    def __init__(self, state_dict, batch, height, width, *, lora, lora_alpha=1.0, attn_reg_weight=0.01,
                 reg_full_identity=True, lr=1e-4, state=None, state_offset=0, text_grad=False, where='Attention',
                 shared_ehs=False, **kw):
        """where: the LoRA placement (UNET_WHERE); `lora` must hold a pair for every module of lora_module_names(), or be
        None for a frozen UNet (only with a shared `state`: the text encoder trains).
        state / state_offset: a shared dp.FlatTrainState (and the offset of the UNet-LoRA block in it) when the text
        encoder is trained in the same step (clip_train_engine.CLIPTrainEngine); None = a private state.
        text_grad: also produce d loss / d(text embeddings) into `self.d_ehs` (bf16 [16 * B * 77, 800], layer-major rows =
        the layout of `in_ehs`; the first 768 columns are the gradient) for the text encoder's backward.
        shared_ehs: one text embedding for all cross-attention layers (vanilla LoRA): `in_ehs` [1, B, 77, 768], `d_ehs`
        bf16 [B * 77, 800] rounded from the fp32 layer sum `d_ehs_f32` [B * 77, 800]."""
        if where not in UNET_WHERE:
            raise ValueError(f'where: {where!r} is not one of {UNET_WHERE}')
        # the backward (col2im_s2, upsample2x_bwd) undoes exact halvings only: a level of odd size would be misread
        f = 2 ** (len(kw.get('block_out', (320, 640, 1280, 1280))) - 1)
        if height % f or width % f:
            raise ValueError(f'training needs latent sides that are multiples of {f} (images of multiples of {8 * f} '
                             f'pixels); got a {height} x {width} latent')
        self.where = where
        self.shared_ehs = bool(shared_ehs)
        self.use_train_graph = bool(kw.pop('use_graph', True))
        self._ext_state, self._state_off, self.text_grad = state, int(state_offset), bool(text_grad)
        self.tgraph = None
        self._tgraphs = {}
        self._accumulate = False
        super().__init__(state_dict, batch, height, width, lora=lora, lora_alpha=lora_alpha, use_graph=False,
                         act_dtype=BF16, **kw)
        self.attn_reg_weight = attn_reg_weight
        self.reg_full_identity = reg_full_identity
        self.wb = {}
        self._build_lora_state(lora, lr)
        self._build_backward_packs()
        self.alphas_cumprod = self._alphas_cumprod().to(self.dev)
        B, H, W = self.B, self.H, self.W
        self.target = torch.zeros(B, 4, H, W, device=self.dev)
        self.d_eps = torch.zeros(B, 4, H, W, device=self.dev)
        self.loss_mask = torch.ones(B, 1, H, W, device=self.dev)
        self.masks = torch.ones(B, 1, H, W, device=self.dev)
        self.pos = torch.zeros(B, 2, device=self.dev, dtype=torch.int32)
        self.t_i32 = torch.zeros(B, device=self.dev, dtype=torch.int32)
        self.mse = torch.zeros(1, device=self.dev)
        self.loss_out = torch.zeros(2, device=self.dev)       # [total loss, attention loss (NaN when skipped)]
        self.mse_ws = torch.zeros(2 * B, device=self.dev)
        self.x0 = torch.zeros(B, 4, H, W, device=self.dev)

    @staticmethod
    def _alphas_cumprod(n=1000, beta_start=0.00085, beta_end=0.012):
        """SD1.5 scaled-linear schedule (scheduler config of the checkpoint the reference loads, trainer_edlora.py:43)."""
        betas = torch.linspace(beta_start ** 0.5, beta_end ** 0.5, n, dtype=torch.float32) ** 2
        return torch.cumprod(1.0 - betas, dim=0)

    def _alloc_io(self):
        super()._alloc_io()
        if self.shared_ehs:
            self.in_ehs = torch.zeros(1, self.B, self.n_text, self.cross_dim, device=self.dev, dtype=self.ACT)

    def _ehs(self, xidx):
        """the text embedding cross-attention layer xidx reads: its own slice, or the shared one"""
        return self.in_ehs[0 if self.shared_ehs else xidx]

    # ------------------------------------------------------------------------------------------ LoRA state
    def lora_module_names(self):
        """The modules that carry a LoRA, in the order of the reference's module walk (trainer_edlora.py:121-133)."""
        whole = getattr(self, 'where', 'Attention') == 'Transformer2DModel'
        names = []
        for an in self.xattn_names:
            tb = an[:-len('.attn2')]
            tn = tb[:-len('.transformer_blocks.0')]
            if whole:
                names.append(f'{tn}.proj_in')
            for a in ('attn1', 'attn2'):
                for p in _PROJ:
                    names.append(f'{tb}.{a}.{p}')
            if whole:
                names += [tb + _GEGLU, f'{tb}.ff.net.2', f'{tn}.proj_out']
        return names

    @property
    def whole_block(self):
        return self.where == 'Transformer2DModel'

    def _fwd_slot(self, m):
        """module name -> (forward pack key, segment index inside the fused pack)"""
        if m.endswith('.proj_in') or m.endswith('.proj_out'):
            return m, 0
        if m.endswith(_GEGLU):
            return m[:-len(_GEGLU)] + '.ff1', 0
        if m.endswith('.ff.net.2'):
            return m[:-len('.ff.net.2')] + '.ff2', 0
        if '.attn1.' in m:
            tb, p = m.split('.attn1.')
            if p == 'to_out.0':
                return f'{tb}.attn1.out', 0
            return f'{tb}.attn1.qkv', ('to_q', 'to_k', 'to_v').index(p)
        tb, p = m.split('.attn2.')
        if p == 'to_q':
            return f'{tb}.attn2.q', 0
        if p == 'to_out.0':
            return f'{tb}.attn2.out', 0
        return f'{tb}.attn2.kv', ('to_k', 'to_v').index(p)

    def _bwd_key(self, m):
        """key of the transposed (dX) pack that carries module m's LoRA term: the attention projections have packs of their
        own (the forward fuses q|k|v), the other modules share the forward pack's key"""
        return m if ('.attn1.' in m or '.attn2.' in m) else self._fwd_slot(m)[0]

    def _build_lora_state(self, lora, lr):
        mods = self.lora_module_names() if lora is not None else []
        if lora is None and self._ext_state is None:
            raise ValueError('a frozen UNet (lora=None) trains nothing of its own: pass the shared state of the text encoder')
        sizes = []
        for m in mods:
            kd = f'{m}.lora_down.weight'
            if kd not in lora:
                raise ValueError(f'training needs a LoRA pair on every module of `where: {self.where}`; missing {kd}')
            K = lora[kd].reshape(lora[kd].shape[0], -1).shape[1]
            N = lora[f'{m}.lora_up.weight'].shape[0]
            sizes.append((K, N))
        total = sum(4 * (k + n) for k, n in sizes)
        if self._ext_state is not None:
            self.state = self._ext_state
            assert self._state_off + total <= self.state.n, 'shared flat state too small for the UNet LoRA block'
        else:
            self.state = FlatTrainState(0, self.cross_dim, 0, total, lrs=(1e-3, 1e-5, lr), device=self.dev)
        self.lora_views = {}
        rows = []
        off = self._state_off
        keep = []
        for m, (K, N) in zip(mods, sizes):
            D = self.state.params[off:off + 4 * K].view(4, K)
            gD = self.state.grads[off:off + 4 * K].view(4, K)
            off += 4 * K
            U = self.state.params[off:off + 4 * N].view(N, 4)
            gU = self.state.grads[off:off + 4 * N].view(N, 4)
            off += 4 * N
            self.lora_views[m] = (D, U, gD, gU, K, N)
            key, seg = self._fwd_slot(m)
            ent = self.w[key]
            row_off = seg * N
            fdown = ent['lora_down'].data_ptr() + 4 * seg * K * 2
            fup = ent['lora_up'].data_ptr() + row_off * 4 * 4
            bdown = bup = 0
            is_kv = self._is_text_kv(m)
            if not is_kv or self.text_grad:
                # text K / V projections: their input gradient d(ehs) is only needed when the text encoder trains; its
                # width 768 is padded to the GEMM's 160-column tiles (800, zero rows)
                kp = _r(K, 160) if is_kv else K
                bd = torch.zeros(16, N, device=self.dev, dtype=BF16)
                bu = torch.zeros(kp, 4, device=self.dev)
                keep += [bd, bu]
                bdown, bup = bd.data_ptr(), bu.data_ptr()
                self.wb[self._bwd_key(m)] = {'N': kp, 'K': N, 'bias': None, 'lora_down': bd, 'lora_up': bu,
                                             'lora_seg': kp}
            rows.append([D.data_ptr(), U.data_ptr(), K, N, fdown, fup, bdown, bup])
        self._lora_keep = keep
        self.lora_table = torch.tensor(rows, dtype=torch.int64, device=self.dev)
        if lora is not None:
            self.load_lora_state_dict(lora)

    def _is_text_kv(self, m):
        return m.endswith('attn2.to_k') or m.endswith('attn2.to_v')

    def _frozen_bwd_entry(self, m):
        """dX pack entry of an attention projection of a frozen UNet: no LoRA term (W is filled by _build_backward_packs)"""
        key, _ = self._fwd_slot(m)
        ent = self.w[key]
        N = ent['N'] // (3 if key.endswith('.qkv') else 2 if key.endswith('.kv') else 1)
        K = ent['K']
        return {'N': _r(K, 160) if self._is_text_kv(m) else K, 'K': N, 'bias': None}

    def refresh_lora(self):
        """Re-pack the flat LoRA parameters into the GEMM operand layouts (after load / optimiser step); nothing for a
        frozen UNet."""
        if self.lora_views:
            ops.lora_pack(self.lora_table, self.lora_table.shape[0], self.lora_alpha)

    def _up_perm(self, m):
        """row permutation natural -> flat of module m's LoRA up (None = identity): the GEGLU projection's flat up is in the
        packed row order of its GEMM"""
        return geglu_perm(self.lora_views[m][5]).to(self.dev) if m.endswith(_GEGLU) else None

    def load_lora_state_dict(self, lora):
        """reference checkpoint tensors (down [r, K] or [r, K, 1, 1], up [N, r] or [N, r, 1, 1], rank r <= 4) -> the flat
        state, then re-pack."""
        for m, (D, U, _, _, K, N) in self.lora_views.items():
            d = lora[f'{m}.lora_down.weight'].detach().to(self.dev, F32).reshape(-1, K)
            u = lora[f'{m}.lora_up.weight'].detach().to(self.dev, F32).reshape(N, -1)
            perm = self._up_perm(m)
            if perm is not None:
                u = u[perm]
            D.zero_()
            U.zero_()
            D[:d.shape[0]] = d
            U[:, :u.shape[1]] = u
        self.refresh_lora()

    def _natural(self, m, U):
        perm = self._up_perm(m)
        if perm is None:
            return U.clone()
        out = torch.empty_like(U)
        out[perm] = U
        return out

    def lora_state_dict(self):
        """{f'{module}.lora_down.weight' [4,K], f'{module}.lora_up.weight' [N,4]} (trainer_edlora.py:371-378 keys); the 1x1
        convs proj_in / proj_out as [4, K, 1, 1] / [N, 4, 1, 1] (the reference wraps a Conv2d there)."""
        out = {}
        for m, (D, U, _, _, _, _) in self.lora_views.items():
            d, u = D.clone(), self._natural(m, U)
            if m.endswith('.proj_in') or m.endswith('.proj_out'):
                d, u = d[:, :, None, None], u[:, :, None, None]
            out[f'{m}.lora_down.weight'] = d
            out[f'{m}.lora_up.weight'] = u
        return out

    def lora_grad_dict(self):
        return {m: (gD.clone(), self._natural(m, gU)) for m, (_, _, gD, gU, _, _) in self.lora_views.items()}

    # ------------------------------------------------------------------------------------------ backward packs
    def _build_backward_packs(self):
        def lin(key):
            W = self.w[key]['W']
            return {'W': W.t().contiguous(), 'N': W.shape[1], 'K': W.shape[0], 'bias': None}

        def conv3(key):
            W = self.w[key]['W']
            cout, cin = W.shape[0], W.shape[1] // 9
            Wb = W.view(cout, 3, 3, cin).flip(1, 2).permute(3, 1, 2, 0).reshape(cin, 9 * cout).contiguous()
            return {'W': Wb, 'N': cin, 'K': 9 * cout, 'bias': None}

        for key in list(self.w):
            if key in self.wb:
                continue            # a LoRA'd module's own pack (_build_lora_state): its weight is filled in below
            if key.endswith('.conv1') or key.endswith('.conv2') or key.endswith('upsamplers.0.conv'):
                self.wb[key] = conv3(key)
            elif key.endswith('.conv_shortcut') or key.endswith('.proj_in') or key.endswith('.proj_out') or \
                    key.endswith('.ff1') or key.endswith('.ff2') or key.endswith('downsamplers.0.conv'):
                self.wb[key] = lin(key)
        for m in self.lora_module_names():
            bk = self._bwd_key(m)
            if bk not in self.wb:
                if self.lora_views or (self._is_text_kv(m) and not self.text_grad):
                    continue
                self.wb[bk] = self._frozen_bwd_entry(m)
            key, seg = self._fwd_slot(m)
            W = self.w[key]['W']
            N = self.wb[bk]['K']
            Wt = W[seg * N:(seg + 1) * N].t()
            if self.wb[bk]['N'] != Wt.shape[0]:                # padded output width (text K / V: 768 -> 800)
                Wp = torch.zeros(self.wb[bk]['N'], N, device=self.dev, dtype=W.dtype)
                Wp[:Wt.shape[0]] = Wt
                Wt = Wp
            self.wb[bk]['W'] = Wt.contiguous()
        self.d_ehs = self.d_ehs_f32 = None
        if self.text_grad:
            rows = (1 if self.shared_ehs else len(self.xattn_names)) * self.B * self.n_text
            self.d_ehs = torch.zeros(rows, _r(self.cross_dim, 160), device=self.dev, dtype=BF16)
            if self.shared_ehs:
                self.d_ehs_f32 = torch.zeros(rows, _r(self.cross_dim, 160), device=self.dev, dtype=F32)

    # ------------------------------------------------------------------------------------------ buffers
    def tb(self, tag, shape, dtype=BF16, zero=False):
        """persistent (saved-for-backward / gradient) buffer, unique per tag"""
        return self.buf('T.' + tag, shape, dtype, zero)

    def _lg_ws(self, M, K, N):
        need = 128 * 4 * (K + N)            # mos_lora_grad: at most 128 row slabs, one partial [4K + 4N] each
        cur = getattr(self, '_lg_buf', None)
        if cur is None or cur.numel() < need:
            self._lg_buf = torch.empty(max(need, 1 << 20), device=self.dev)
        return self._lg_buf

    def _gnws(self):
        return self.buf('gn_bwd_ws', (self.B * 1184 * 128,), F32)

    # ------------------------------------------------------------------------------------------ forward blocks
    def resnet_train(self, name, x, out, h, w, cin, cout):
        B = self.B
        HW = h * w
        M = B * HW
        res = x
        has_sc = name + '.conv_shortcut' in self.w
        if has_sc:
            sc = self.buf('rn_sc', (M, cout))
            self.gemm(x, self.w[name + '.conv_shortcut'], sc, M=M, lda=x.stride(0))
            res = sc
        n1 = self.buf('rn_n', (M, cin))
        self.groupnorm(x, name + '.norm1', n1, HW=HW, C=cin, eps=1e-5, silu=True)
        h1 = self.tb(name + '.h1', (M, cout))
        tbp = self.tproj[:, self.temb_off[name]:]
        self.gemm(n1, self.w[name + '.conv1'], h1, M=M, conv=(B, h, w, cin), bias_batch=tbp, rows_per_batch=HW)
        n2 = self.buf('rn_n2', (M, cout))
        self.groupnorm(h1, name + '.norm2', n2, HW=HW, C=cout, eps=1e-5, silu=True)
        self.gemm(n2, self.w[name + '.conv2'], out, M=M, conv=(B, h, w, cout), residual=res)
        self.trace.append(('resnet', name, x, out, h, w, cin, cout, h1))
        return out

    def resnet_bwd(self, e, dOut):
        _, name, x, out, h, w, cin, cout, h1 = e
        B = self.B
        HW = h * w
        M = B * HW
        d_n2 = self.buf('g_rn_a', (M, cout))
        self.gemm(dOut, self.wb[name + '.conv2'], d_n2, M=M, conv=(B, h, w, cout), lda=dOut.stride(0))
        g2, b2 = self.w[name + '.norm2']
        d_h1 = self.buf('g_rn_b', (M, cout))
        ops.groupnorm_bwd(h1, d_n2, g2, b2, d_h1, self._gnws(), B=B, HW=HW, C=cout, eps=1e-5, silu=True)
        d_n1 = self.buf('g_rn_c', (M, cin))
        self.gemm(d_h1, self.wb[name + '.conv1'], d_n1, M=M, conv=(B, h, w, cout))
        add = dOut
        if name + '.conv_shortcut' in self.w:
            add = self.buf('g_rn_d', (M, cin))
            self.gemm(dOut, self.wb[name + '.conv_shortcut'], add, M=M, lda=dOut.stride(0))
        g1, b1 = self.w[name + '.norm1']
        dX = self.tb('g.' + name, (M, cin))
        ops.groupnorm_bwd(x, d_n1, g1, b1, dX, self._gnws(), B=B, HW=HW, C=cin, eps=1e-5, silu=True, add=add,
                          ldx=x.stride(0), ldadd=add.stride(0))
        return dX

    def _cross_kv_train(self, tbn, ehs_layer, C, xidx):
        B, T = self.B, self.n_text
        d = C // self.heads
        BH = B * self.heads
        Kc = self.tb(f'Kc{xidx}', (BH, T, _r(d, 64)), zero=True)
        Vc = self.tb(f'Vc{xidx}', (BH, T, _r(d, 64)), zero=True)
        A = ehs_layer.reshape(B * T, self.cross_dim)
        self.gemm(A, self.w[tbn + '.attn2.kv'], None, M=B * T,
                  heads=self._heads([Kc, Vc], [MOS_SEG_ROWS, MOS_SEG_ROWS], [T, T], C, T))
        Kct = self.tb(f'Kct{xidx}', (BH, _r(d, 16), _r(T, 8)), zero=True)
        Vct = self.tb(f'Vct{xidx}', (BH, _r(d, 16), _r(T, 8)), zero=True)
        ops.heads_transpose(Kc, Kct)
        ops.heads_transpose(Vc, Vct)
        return Kc, Vc, Kct, Vct

    def _gemm_in(self, tn, tag, shape):
        """input of proj_in / ff.net.0.proj / ff.net.2 / proj_out: kept for the LoRA gradient when those modules carry a
        LoRA (`where: Transformer2DModel`), a scratch buffer otherwise"""
        return self.tb(f'{tn}.{tag}', shape) if self.whole_block else self.buf('tr_' + tag, shape)

    def transformer_train(self, tn, x, out, h, w, C, xidx):
        B, Hh = self.B, self.heads
        N = h * w
        M = B * N
        d = C // Hh
        BH = B * Hh
        dp, dv = _r(d, 64), _r(d, 16)
        tbn = tn + '.transformer_blocks.0'
        S = {}
        gn = self._gemm_in(tn, 'gn', (M, C))
        self.groupnorm(x, tn + '.norm', gn, HW=N, C=C, eps=1e-6, silu=False)
        t0 = self.tb(tn + '.t0', (M, C))
        self.gemm(gn, self.w[tn + '.proj_in'], t0, M=M)
        # --- attn1
        ln1 = self.tb(tn + '.ln1', (M, C))
        self.layernorm(t0, tbn + '.norm1', ln1, M=M, C=C)
        Q = self.tb(tn + '.Q1', (BH, N, dp), zero=True)
        K = self.tb(tn + '.K1', (BH, N, dp), zero=True)
        V = self.tb(tn + '.V1', (BH, N, dp), zero=True)
        self.gemm(ln1, self.w[tbn + '.attn1.qkv'], None, M=M,
                  heads=self._heads([Q, K, V], [MOS_SEG_ROWS] * 3, [N, N, N], C, N))
        Vt = self.buf('Vt', (BH, dv, _r(N, 8)), zero=True)
        ops.heads_transpose(V, Vt)
        ao1 = self.tb(tn + '.ao1', (M, C))
        lse1 = self.tb(tn + '.lse1', (BH, N), F32)
        ops.attention_train(Q, K, Vt, ao1.view(B, N, C), lse1, batch=B, heads=Hh, head_dim=d, nq=N, nk=N)
        t1 = self.tb(tn + '.t1', (M, C))
        self.gemm(ao1, self.w[tbn + '.attn1.out'], t1, M=M, residual=t0)
        # --- attn2 (layer-wise text embedding, edlora.py:129-131)
        ln2 = self.tb(tn + '.ln2', (M, C))
        self.layernorm(t1, tbn + '.norm2', ln2, M=M, C=C)
        Q2 = self.tb(tn + '.Q2', (BH, N, dp), zero=True)
        self.gemm(ln2, self.w[tbn + '.attn2.q'], None, M=M, heads=self._heads([Q2], [MOS_SEG_ROWS], [N], C, N))
        Kc, Vc, Kct, Vct = self.kvt[xidx]
        ao2 = self.tb(tn + '.ao2', (M, C))
        lse2 = self.tb(tn + '.lse2', (BH, N), F32)
        pcols = self.tb(tn + '.pcols', (BH, N, 2), F32) if self.attn_reg_weight is not None else None
        ops.attention_train(Q2, Kc, Vct, ao2.view(B, N, C), lse2, batch=B, heads=Hh, head_dim=d, nq=N, nk=self.n_text,
                            pcols=pcols, pos=self.pos if pcols is not None else None)
        t2 = self.tb(tn + '.t2', (M, C))
        self.gemm(ao2, self.w[tbn + '.attn2.out'], t2, M=M, residual=t1)
        # --- feed-forward (un-fused GEGLU: the pre-activation is kept for backward)
        ln3 = self._gemm_in(tn, 'ln', (M, C))
        self.layernorm(t2, tbn + '.norm3', ln3, M=M, C=C)
        z = self.tb(tn + '.z', (M, 8 * C))
        self.gemm(ln3, self.w[tbn + '.ff1'], z, M=M)
        ff = self._gemm_in(tn, 'ff', (M, 4 * C))
        ops.geglu_fwd(z, ff, M=M, H=4 * C)
        t3 = self._gemm_in(tn, 't3', (M, C))
        self.gemm(ff, self.w[tbn + '.ff2'], t3, M=M, residual=t2)
        self.gemm(t3, self.w[tn + '.proj_out'], out, M=M, residual=x)
        S.update(t0=t0, ln1=ln1, Q=Q, K=K, V=V, ao1=ao1, lse1=lse1, t1=t1, ln2=ln2, Q2=Q2, ao2=ao2, lse2=lse2,
                 pcols=pcols, t2=t2, z=z, gn=gn, ln3=ln3, ff=ff, t3=t3)
        self.trace.append(('transformer', tn, x, out, h, w, C, xidx, S))
        self.pcols_by_layer[xidx] = (pcols, N)
        return out

    def _lora_grad(self, m, x, dy, M, ldx=None, lddy=None):
        if not self.lora_views:
            return                  # frozen UNet: no LoRA gradient
        D, U, gD, gU, K, N = self.lora_views[m]
        ops.lora_grad(x, dy, D, U, self.lora_alpha, self._lg_ws(M, K, N), gD, gU, M=M, K=K, N=N, ldx=ldx, lddy=lddy,
                      accumulate=self._accumulate)

    def _gemm_f32(self, A, ent, out, *, M, lda, accumulate):
        """out (fp32) = [out +] A @ ent^T (+ its LoRA term): one launch, no split-K (the fp32 output path takes none)"""
        kw = {}
        if 'lora_down' in ent:
            kw = dict(lora_down=ent['lora_down'], lora_up=ent['lora_up'], lora_seg=ent['lora_seg'])
        ops.gemm(A, ent['W'], out, M=M, lda=lda, out_f32=True, accumulate=accumulate, **kw)
        self.launches += 1

    def _attn_bwd(self, Q, K, V, ao, lse, dO, dq, dk, dv, N, nk, d, pcols=None, gcols=None):
        B, Hh = self.B, self.heads
        BH = B * Hh
        dv_ = _r(d, 16)
        Qt = self.buf('g_Qt', (BH, dv_, _r(N, 8)), zero=True)
        dOt = self.buf('g_dOt', (BH, dv_, _r(N, 8)), zero=True)
        Kt = self.buf(f'g_Kt{nk}', (BH, dv_, _r(nk, 8)), zero=True)
        ops.heads_transpose(Q, Qt)
        ops.heads_transpose(dO, dOt)
        ops.heads_transpose(K, Kt)
        delta = self.buf('g_delta', (BH, N), F32)
        ops.attn_delta(dO, ao, delta, batch=B, heads=Hh, head_dim=d, N=N, ldo=ao.stride(0), pcols=pcols, gcols=gcols)
        ops.attention_bwd(Q, K, V, dO, Qt, Kt, dOt, lse, delta, dq, dk, dv, batch=B, heads=Hh, head_dim=d, nq=N,
                          nk=nk, gcols=gcols, pos=self.pos if gcols is not None else None, lddq=dq.stride(0),
                          lddk=dk.stride(0), lddv=dv.stride(0))

    def transformer_bwd(self, e, dOut):
        _, tn, x, out, h, w, C, xidx, S = e
        B, Hh = self.B, self.heads
        N = h * w
        M = B * N
        T = self.n_text
        d = C // Hh
        BH = B * Hh
        dp = _r(d, 64)
        tbn = tn + '.transformer_blocks.0'
        a1, a2 = tbn + '.attn1.', tbn + '.attn2.'
        whole = self.whole_block
        # proj_out, feed-forward (with `where: Transformer2DModel` their dX packs carry the LoRA term)
        if whole:
            self._lora_grad(tn + '.proj_out', S['t3'], dOut, M, lddy=dOut.stride(0))
        d_t3 = self.buf('g_t3', (M, C))
        self.gemm(dOut, self.wb[tn + '.proj_out'], d_t3, M=M, lda=dOut.stride(0))
        if whole:
            self._lora_grad(tbn + '.ff.net.2', S['ff'], d_t3, M)
        d_y = self.buf('g_ff', (M, 4 * C))
        self.gemm(d_t3, self.wb[tbn + '.ff2'], d_y, M=M)
        d_z = self.buf('g_z', (M, 8 * C))
        ops.geglu_bwd(S['z'], d_y, d_z, M=M, H=4 * C)
        if whole:           # d_z and the flat LoRA up are both in the packed (interleaved) row order
            self._lora_grad(tbn + _GEGLU, S['ln3'], d_z, M)
        d_ln = self.buf('g_ln', (M, C))
        self.gemm(d_z, self.wb[tbn + '.ff1'], d_ln, M=M)
        d_t2 = self.buf('g_t2', (M, C))
        ops.layernorm_bwd(S['t2'], d_ln, self.w[tbn + '.norm3'][0], d_t2, M=M, C=C, add=d_t3)
        # attn2
        self._lora_grad(a2 + 'to_out.0', S['ao2'], d_t2, M)
        dO = self.buf('g_dO', (BH, N, dp), zero=True)
        self.gemm(d_t2, self.wb[a2 + 'to_out.0'], None, M=M, heads=self._heads([dO], [MOS_SEG_ROWS], [N], C, N))
        Kc, Vc, Kct, Vct = self.kvt[xidx]
        dq = self.buf('g_dq', (M, C))
        dkv = self.buf('g_dkv', (B * T, 2 * C))
        gcols = self.gcols_by_layer.get(xidx)
        self._attn_bwd(S['Q2'], Kc, Vc, S['ao2'], S['lse2'], dO, dq, dkv[:, :C], dkv[:, C:], N, T, d,
                       pcols=S['pcols'] if gcols is not None else None, gcols=gcols)
        ehs = self._ehs(xidx).reshape(B * T, self.cross_dim)
        self._lora_grad(a2 + 'to_q', S['ln2'], dq, M)
        self._lora_grad(a2 + 'to_k', ehs, dkv[:, :C], B * T, lddy=2 * C)
        self._lora_grad(a2 + 'to_v', ehs, dkv[:, C:], B * T, lddy=2 * C)
        if self.d_ehs_f32 is not None:  # shared embedding: the same two products, added to the fp32 layer sum
            self._gemm_f32(dkv[:, :C], self.wb[a2 + 'to_k'], self.d_ehs_f32, M=B * T, lda=2 * C,
                           accumulate=not self._dehs_first)
            self._gemm_f32(dkv[:, C:], self.wb[a2 + 'to_v'], self.d_ehs_f32, M=B * T, lda=2 * C, accumulate=True)
            self._dehs_first = False
        elif self.d_ehs is not None:    # d(text embedding of layer xidx) = dK (W_k + a U_k D_k) + dV (W_v + a U_v D_v)
            dst = self.d_ehs[xidx * B * T:(xidx + 1) * B * T]
            self.gemm(dkv[:, :C], self.wb[a2 + 'to_k'], dst, M=B * T, lda=2 * C)
            self.gemm(dkv[:, C:], self.wb[a2 + 'to_v'], dst, M=B * T, lda=2 * C, residual=dst)
        self.gemm(dq, self.wb[a2 + 'to_q'], d_ln, M=M)
        d_t1 = self.buf('g_t1', (M, C))
        ops.layernorm_bwd(S['t1'], d_ln, self.w[tbn + '.norm2'][0], d_t1, M=M, C=C, add=d_t2)
        # attn1
        self._lora_grad(a1 + 'to_out.0', S['ao1'], d_t1, M)
        self.gemm(d_t1, self.wb[a1 + 'to_out.0'], None, M=M, heads=self._heads([dO], [MOS_SEG_ROWS], [N], C, N))
        dqkv = self.buf('g_dqkv', (M, 3 * C))
        self._attn_bwd(S['Q'], S['K'], S['V'], S['ao1'], S['lse1'], dO, dqkv[:, :C], dqkv[:, C:2 * C], dqkv[:, 2 * C:],
                       N, N, d)
        for s, p in enumerate(('to_q', 'to_k', 'to_v')):
            sl = dqkv[:, s * C:(s + 1) * C]
            self._lora_grad(a1 + p, S['ln1'], sl, M, lddy=3 * C)
            self.gemm(sl, self.wb[a1 + p], d_ln, M=M, lda=3 * C, residual=d_ln if s > 0 else None)
        d_t0 = self.buf('g_t0', (M, C))
        ops.layernorm_bwd(S['t0'], d_ln, self.w[tbn + '.norm1'][0], d_t0, M=M, C=C, add=d_t1)
        if whole:
            self._lora_grad(tn + '.proj_in', S['gn'], d_t0, M)
        d_gn = self.buf('g_gn', (M, C))
        self.gemm(d_t0, self.wb[tn + '.proj_in'], d_gn, M=M)
        g, b = self.w[tn + '.norm']
        dX = self.tb('g.' + tn, (M, C))
        ops.groupnorm_bwd(x, d_gn, g, b, dX, self._gnws(), B=B, HW=N, C=C, eps=1e-6, silu=False, add=dOut,
                          ldx=x.stride(0), ldadd=dOut.stride(0))
        return dX

    # ------------------------------------------------------------------------------------------ forward
    def _run_train(self):
        B, H, W = self.B, self.H, self.W
        nb = len(self.block_out)
        self.launches = 0
        self.trace = []
        self.pcols_by_layer = {}
        self.gcols_by_layer = {}
        self._time()
        self.kvt = {}
        chans = self._xattn_channels()
        for xidx, (an, C) in enumerate(zip(self.xattn_names, chans)):
            self.kvt[xidx] = self._cross_kv_train(an[:-len('.attn2')], self._ehs(xidx), C, xidx)
        si = 0
        x = self._skip_slot(si)
        ops.conv_in(self.in_latents, self.w['conv_in'][0], self.w['conv_in'][1], x, ldy=x.stride(0))
        si += 1
        h, w, cin = H, W, self.block_out[0]
        xi = 0
        for i, c in enumerate(self.block_out):
            has_attn = i < nb - 1
            for j in range(self.layers):
                slot = self._skip_slot(si)
                si += 1
                M = B * h * w
                rn = f'down_blocks.{i}.resnets.{j}'
                if has_attn:
                    r = self.tb(rn + '.out', (M, c))
                    self.resnet_train(rn, x, r, h, w, cin, c)
                    self.transformer_train(f'down_blocks.{i}.attentions.{j}', r, slot, h, w, c, xi)
                    xi += 1
                else:
                    self.resnet_train(rn, x, slot, h, w, cin, c)
                x, cin = slot, c
            if has_attn:
                slot = self._skip_slot(si)
                si += 1
                Mo = B * (h // 2) * (w // 2)
                col = self.buf('im2col', (Mo, 9 * c))
                ops.im2col_s2(x, col, B=B, H=h, W=w, C=c, ldx=x.stride(0))
                self.gemm(col, self.w[f'down_blocks.{i}.downsamplers.0.conv'], slot, M=Mo)
                self.trace.append(('down', f'down_blocks.{i}.downsamplers.0.conv', x, slot, h, w, c))
                h, w = h // 2, w // 2
                x = slot
        c = self.block_out[-1]
        M = B * h * w
        r = self.tb('mid.r0', (M, c))
        self.resnet_train('mid_block.resnets.0', x, r, h, w, c, c)
        r2 = self.tb('mid.r1', (M, c))
        self.transformer_train('mid_block.attentions.0', r, r2, h, w, c, xi)
        xi += 1
        k = 0
        dst = self.cat[0][:, :self.cat_ch[0][0]]
        self.resnet_train('mid_block.resnets.1', r2, dst, h, w, c, c)
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
                    nxt = self.tb('final', (M, c))
                elif last_in_block:
                    nxt = self.tb(f'up_pre{i}', (M, c))
                else:
                    nxt = self.cat[k + 1][:, :self.cat_ch[k + 1][0]]
                rn = f'up_blocks.{i}.resnets.{j}'
                if has_attn:
                    r = self.tb(rn + '.out', (M, c))
                    self.resnet_train(rn, xin, r, h, w, ch + cs, c)
                    self.transformer_train(f'up_blocks.{i}.attentions.{j}', r, nxt, h, w, c, xi)
                    xi += 1
                else:
                    self.resnet_train(rn, xin, nxt, h, w, ch + cs, c)
                k += 1
                if last_in_block and not final:
                    up = self.buf('up_x', (B * 4 * h * w, c))
                    ops.upsample2x(nxt, up, B=B, H=h, W=w, C=c, ldx=nxt.stride(0))
                    dst = self.cat[k][:, :self.cat_ch[k][0]]
                    self.gemm(up, self.w[f'up_blocks.{i}.upsamplers.0.conv'], dst, M=B * 4 * h * w,
                              conv=(B, 2 * h, 2 * w, c))
                    self.trace.append(('up', f'up_blocks.{i}.upsamplers.0.conv', nxt, dst, h, w, c))
                    h, w = 2 * h, 2 * w
        M = B * h * w
        c0 = self.block_out[0]
        fin = self.tb('final', (M, c0))
        fn = self.buf('final_n', (M, c0))
        self.groupnorm(fin, 'conv_norm_out', fn, HW=h * w, C=c0, eps=1e-5, silu=True)
        ops.conv_out(fn, self.w['conv_out'][0], self.w['conv_out'][1], self.out_eps, B=B, H=h, W=w, C=c0)
        self._final = (fin, h, w, c0)

    # ------------------------------------------------------------------------------------------ loss
    def _loss(self):
        B = self.B
        ops.masked_mse(self.out_eps, self.target, self.loss_mask, self.mse_ws, self.mse, self.d_eps)
        if self.attn_reg_weight is None:
            self.loss_out[0:1].copy_(self.mse)
            self.loss_out[1:2].zero_()
            return
        groups = {}
        for xidx in sorted(self.pcols_by_layer):
            pc, N = self.pcols_by_layer[xidx]
            groups.setdefault(N, []).append((xidx, pc))
        order = sorted(groups, reverse=True)
        stats = self.buf('reg_stats', (len(order), 8), F32)
        cms = []
        for g, N in enumerate(order):
            res = int(math.isqrt(N))
            cm = self.buf(f'reg_cm{N}', (B, N, 2), F32)
            ops.attn_reg_group([pc for _, pc in groups[N]], self.masks, cm, stats[g], B=B, heads=self.heads, res=res,
                               full_identity=self.reg_full_identity, weight=self.attn_reg_weight)
            cms.append((cm, res))
        ops.attn_reg_total(self.mse, stats, self.loss_out)
        for g, N in enumerate(order):
            cm, res = cms[g]
            gc = self.buf(f'reg_g{N}', (B, N, 2), F32)
            ops.attn_reg_grad(cm, self.masks, stats, gc, B=B, res=res, full_identity=self.reg_full_identity,
                              weight=self.attn_reg_weight, group=g, L=len(groups[N]), heads=self.heads)
            for xidx, _ in groups[N]:
                self.gcols_by_layer[xidx] = gc

    # ------------------------------------------------------------------------------------------ backward
    def _deposit(self, grads, x, g):
        k = _key(x)
        if k in self._cat_keys:
            ch, cs = self._cat_keys[k]
            self._deposit(grads, x[:, :ch], g[:, :ch])
            self._deposit(grads, x[:, ch:], g[:, ch:])
            return
        if k in grads:
            ops.add_rows(grads[k], g, M=x.shape[0], C=x.shape[1], ldx=grads[k].stride(0), ldr=g.stride(0))
        else:
            grads[k] = g

    def _backward(self):
        B = self.B
        self._cat_keys = {_key(c): cc for c, cc in zip(self.cat, self.cat_ch)}
        fin, h, w, c0 = self._final
        M = B * h * w
        d_fn = self.buf('g_fn', (M, c0))
        ops.conv_out_bwd(self.d_eps, self.w['conv_out'][0], d_fn, B=B, H=h, W=w, C=c0)
        g, b = self.w['conv_norm_out']
        d_fin = self.tb('g.final', (M, c0))
        ops.groupnorm_bwd(fin, d_fn, g, b, d_fin, self._gnws(), B=B, HW=h * w, C=c0, eps=1e-5, silu=True)
        grads = {_key(fin): d_fin}
        self._dehs_first = True
        for e in reversed(self.trace):
            kind = e[0]
            if kind == 'resnet':
                dOut = grads.pop(_key(e[3]))
                self._deposit(grads, e[2], self.resnet_bwd(e, dOut))
            elif kind == 'transformer':
                dOut = grads.pop(_key(e[3]))
                self._deposit(grads, e[2], self.transformer_bwd(e, dOut))
            elif kind == 'down':
                _, key, x, slot, h, w, c = e
                dOut = grads.pop(_key(slot))
                Mo = B * (h // 2) * (w // 2)
                dcol = self.buf('g_col', (Mo, 9 * c))
                self.gemm(dOut, self.wb[key], dcol, M=Mo, lda=dOut.stride(0))
                dX = self.tb('g.' + key, (B * h * w, c))
                ops.col2im_s2(dcol, dX, B=B, H=h, W=w, C=c)
                self._deposit(grads, x, dX)
            elif kind == 'up':
                _, key, x, dst, h, w, c = e
                dOut = grads.pop(_key(dst))
                d_up = self.buf('g_up', (B * 4 * h * w, c))
                self.gemm(dOut, self.wb[key], d_up, M=B * 4 * h * w, conv=(B, 2 * h, 2 * w, c), lda=dOut.stride(0))
                dX = self.tb('g.' + key, (B * h * w, c))
                ops.upsample2x_bwd(d_up, dX, B=B, H=h, W=w, C=c)
                self._deposit(grads, x, dX)
        self._leftover = grads      # only the conv_in output gradient remains (the latents need no gradient)
        if self.d_ehs_f32 is not None:  # the fp32 layer sum -> bf16, once (a one-slice "split-K" reduction)
            ops.splitk_finalize(self.d_ehs_f32, 1, self.d_ehs.shape[0], self.d_ehs.shape[1], self.d_ehs)
            self.launches += 1

    # ------------------------------------------------------------------------------------------ public API
    def attach_text_engine(self, text_engine):
        """Run the text encoder in the same (captured) step: `text_engine` (over 16 * B layer-major sequences, B with
        shared_ehs) writes its last hidden state straight into `in_ehs` before the UNet forward.  With text_grad=True it is a
        clip_train_engine.CLIPTrainEngine that consumes `d_ehs` after the UNet backward; with text_grad=False a frozen
        clip_engine.CLIPTextEngine that runs its forward only."""
        assert text_engine.n_seq == (1 if self.shared_ehs else len(self.xattn_names)) * self.B
        assert not self.text_grad or hasattr(text_engine, 'backward'), "text_grad needs a training text engine"
        self.text = text_engine
        self._tgraphs = {}

    def forward_backward(self, latents, noise, timesteps, ehs_layers, masks, loss_mask=None, token_pos=None,
                         accumulate=False, text_ids=None):
        """One forward + loss + backward.  latents (x0) / noise fp32 [B,4,H,W]; timesteps int [B]; ehs_layers bf16
        [16,B,77,768] (shared_ehs: [B,77,768]); masks / loss_mask [B,1,H,W] (trainer_edlora.py:246-252); token_pos: B pairs of concept-token
        positions (:270-279).  Returns the device tensor [total loss, attention loss]."""
        self.t_i32.copy_(timesteps.to(self.dev, torch.int32))
        self.in_t.copy_(timesteps.to(self.dev, F32))
        if getattr(self, 'text', None) is not None:
            self.text.set_ids(text_ids)              # layer-major [16 * B, 77] token ids ([B, 77] with shared_ehs)
        else:
            self.in_ehs.copy_(ehs_layers)
        self.target.copy_(noise)                                     # prediction_type 'epsilon' (:241-242)
        self.masks.copy_(masks)
        self.loss_mask.copy_(masks if loss_mask is None else loss_mask)
        if token_pos is not None:
            self.pos.copy_(torch.as_tensor(token_pos, dtype=torch.int32))
        self.x0.copy_(latents)
        self._accumulate = bool(accumulate)
        if not self.use_train_graph:
            self._step()
            return self.loss_out
        self.tgraph = self._tgraphs.get(self._accumulate)
        if self.tgraph is None:
            # warm-up (allocates every saved-activation / gradient buffer, sets kernel attributes), then capture the
            # whole forward + loss + backward (~2500 launches) in one CUDA graph
            saved = self.state.grads.clone() if self._accumulate else None   # the warm-up run must not count
            torch.cuda.synchronize()
            s = torch.cuda.Stream()
            s.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(s):
                self._step()
            torch.cuda.current_stream().wait_stream(s)
            torch.cuda.synchronize()
            self.tgraph = torch.cuda.CUDAGraph()
            with torch.cuda.graph(self.tgraph):
                self._step()
            self._tgraphs[self._accumulate] = self.tgraph
            if saved is not None:
                self.state.grads.copy_(saved)
        self.tgraph.replay()
        return self.loss_out

    def _step(self):
        text = getattr(self, 'text', None)
        if text is not None:          # text encoder forward: last hidden states -> in_ehs (same layout, no copy)
            if self.text_grad:
                text.forward_train(out=self.in_ehs.view(-1, self.cross_dim))
            else:
                text.encode(self.in_ehs.view(-1, self.cross_dim))
        ops.add_noise(self.x0, self.target, self.t_i32, self.alphas_cumprod, self.in_latents)
        self._run_train()
        self._loss()
        self._backward()
        if text is not None and self.text_grad:          # ... and its backward from d(in_ehs)
            text.backward(self.d_ehs, accumulate=self._accumulate)

    def optimizer_step(self, grad_scale=1.0):
        from .dp import optimizer_step
        optimizer_step(self.state, grad_scale)
        self.refresh_lora()
