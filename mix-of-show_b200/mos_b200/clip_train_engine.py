"""CLIPTrainEngine — the text-encoder half of one ED-LoRA training step on the GPU: forward with saved activations and the
backward that turns d(last_hidden_state) into the gradients of the NEW-CONCEPT EMBEDDING ROWS and of the CLIPAttention LoRA
(`where: CLIPAttention`, q/k/v/out_proj of all 12 layers), built only from libmos_sm100 kernels.

Reference: `encoder_hidden_states = self.text_encoder(text_input_ids)[0]` at mixofshow/pipelines/trainer_edlora.py:220-234
reached by `accelerator.backward(loss)` (train_edlora.py:120-123); parameter groups 1 and 2 of trainer_edlora.py:82-118
(embedding lr 1e-3, text-encoder LoRA lr 1e-5).  All base weights are frozen (:73-76), so the backward produces activation
gradients (tensor-core GEMMs on transposed weight packs with the LoRA term fused, causal flash-attention backward,
LayerNorm / quick-GELU backward), the rank-4 LoRA gradients and the embedding-row gradients, all written into the SAME flat
fp32 buffer as the UNet LoRA gradients (dp.FlatTrainState) so that the data-parallel step keeps its single all-reduce.

Sequence order: the 16 layer-wise prompts of a sample are laid out LAYER-MAJOR (sequence index = layer * B + sample), so
the engine's output [16 * B * 77, 768] IS the UNet engine's `in_ehs` [16, B, 77, 768] and d(in_ehs) IS this engine's output
gradient: no gather / scatter between the two engines.

With `where: CLIPEncoderLayer` (trainer_edlora.py:100-112) mlp.fc1 / mlp.fc2 of every layer are trained too.

Either group may be frozen on its own (the `enable_tuning` flags of trainer_edlora.py:82-118): with `lora=None` the GEMMs
run plain epilogues and the backward issues no LoRA-gradient launch (it still runs through the frozen layers down to the
embedding rows); with `emb_offset=None` the concept rows are constants of the engine's own token table and the
embedding-row gradient launch is skipped.

Flat parameter layout of a LoRA (padded to the GEMM shapes of clip_engine.py; pads are zero and stay zero: their gradients
are exactly zero, so AdamW never moves them):
    q / k / v : down [4, 768], up [960, 4]   (12 heads of 64 dims run as 80: rows h*80+64 .. h*80+79 are pads)
    out_proj  : down [4, 960] (pad columns as above), up [768, 4]
    mlp.fc1   : down [4, 768], up [3200, 4]  (rows 3072 .. 3199 are pads)
    mlp.fc2   : down [4, 3200] (columns 3072 .. 3199 are pads), up [768, 4]
`lora_state_dict()` / `load_lora_state_dict()` convert to / from the reference's checkpoint tensors ([r, in] / [out, r]).
"""
import torch

from . import ops
from ._lib import MOS_SEG_ROWS
from .clip_engine import BF16, PROJ, CLIPTextEngine, _r

F32 = torch.float32
CLIP_WHERE = ('CLIPAttention', 'CLIPEncoderLayer')


class CLIPTrainEngine(CLIPTextEngine):
    def __init__(self, state_dict, n_seq, *, lora, lora_alpha=1.0, concept_token_ids=(), state=None, emb_offset=0,
                 lora_offset=None, where='CLIPAttention', **kw):
        """lora: {f'{module}.lora_down.weight' [r,768], f'{module}.lora_up.weight' [768,r]} for every q/k/v/out_proj of
        every layer (rank <= 4); None = no LoRA (the text-encoder group is frozen).  concept_token_ids: the new-concept
        rows of the token-embedding table.
        state: dp.FlatTrainState to live in (parameters / gradients are views of it): the embedding rows at
        `emb_offset` (None = the rows are not trained and stay in the token table), the LoRA block at `lora_offset`;
        None = a private state.
        where: the LoRA placement (CLIP_WHERE); `lora` must hold a pair for every module of lora_module_names()."""
        if where not in CLIP_WHERE:
            raise ValueError(f'where: {where!r} is not one of {CLIP_WHERE}')
        self.where = where
        super().__init__(state_dict, n_seq, lora=lora, lora_alpha=lora_alpha, **kw)
        self.concept_ids = [int(i) for i in concept_token_ids]
        R, C = len(self.concept_ids), self.C
        n_lora = self.lora_param_count(self.n_layers, C, self.Ca, where=where, inner=self.I) if lora is not None else 0
        if state is None:
            from .dp import FlatTrainState
            state = FlatTrainState(R, C, n_lora, 0, device=self.dev)
            emb_offset, lora_offset = 0, R * C
        self.state = state
        self.rows_dev = torch.tensor(self.concept_ids, dtype=torch.int32, device=self.dev)
        self.train_rows = emb_offset is not None and R > 0
        self.emb_view = self.emb_grad = None
        if self.train_rows:
            self.emb_view = state.params[emb_offset:emb_offset + R * C].view(R, C)
            self.emb_grad = state.grads[emb_offset:emb_offset + R * C].view(R, C)
            self.emb_view.copy_(self.tok[self.rows_dev.long()])
        self._accumulate = False
        self.wb = {}
        self._build_lora_state(lora, lora_offset)
        self._build_backward_packs()
        self.saved = []

    @staticmethod
    def lora_param_count(n_layers, C, Ca, where='CLIPAttention', inner=3072):
        """floats of the flat LoRA block (rank-4 slots, pads included)"""
        n = 3 * (4 * C + 4 * Ca) + (4 * Ca + 4 * C)
        if where == 'CLIPEncoderLayer':
            Ip = _r(inner, 160)
            n += (4 * C + 4 * Ip) + (4 * Ip + 4 * C)
        return n_layers * n

    @staticmethod
    def module_names(n_layers, where='CLIPAttention', prefix='text_model.'):
        """the modules that carry a LoRA, layer by layer (flat-state order)"""
        mlp = ('mlp.fc1', 'mlp.fc2') if where == 'CLIPEncoderLayer' else ()
        return [f'{prefix}encoder.layers.{i}.{p}' for i in range(n_layers)
                for p in tuple('self_attn.' + q for q in PROJ) + mlp]

    # ------------------------------------------------------------------------------------------ LoRA state
    def lora_module_names(self):
        return self.module_names(self.n_layers, self.where, self.pre)

    def _lora_shape(self, m):
        """(K, N) of module m's flat LoRA (down [4, K], up [N, 4])"""
        if m.endswith('out_proj'):
            return self.Ca, self.C
        if m.endswith('fc1'):
            return self.C, self.Ip
        if m.endswith('fc2'):
            return self.Ip, self.C
        return self.C, self.Ca

    def _pad_heads_rows(self, U):        # [heads*d, r] -> [heads*dh, r]
        out = torch.zeros(self.heads, self.dh, U.shape[1], device=self.dev)
        out[:, :self.d] = U.reshape(self.heads, self.d, U.shape[1])
        return out.reshape(self.heads * self.dh, U.shape[1])

    def _pad_heads_cols(self, D):        # [r, heads*d] -> [r, heads*dh]
        out = torch.zeros(D.shape[0], self.heads, self.dh, device=self.dev)
        out[:, :, :self.d] = D.reshape(D.shape[0], self.heads, self.d)
        return out.reshape(D.shape[0], self.heads * self.dh)

    def _build_lora_state(self, lora, off):
        C, Ca, Cp = self.C, self.Ca, self.Cp
        self.lora_views = {}
        rows, keep = [], []
        for m in (self.lora_module_names() if lora is not None else ()):
            kd = f'{m}.lora_down.weight'
            if kd not in lora:
                raise ValueError(f'training needs a LoRA pair on every module of `where: {self.where}`; missing {kd}')
            is_out = m.endswith('out_proj')
            K, N = self._lora_shape(m)
            D = self.state.params[off:off + 4 * K].view(4, K)
            gD = self.state.grads[off:off + 4 * K].view(4, K)
            off += 4 * K
            U = self.state.params[off:off + 4 * N].view(N, 4)
            gU = self.state.grads[off:off + 4 * N].view(N, 4)
            off += 4 * N
            self.lora_views[m] = (D, U, gD, gU, K, N)
            i = int(m.split('.layers.')[1].split('.')[0])
            ent = self.w[i]
            mlp = m.rsplit('.', 1)[1] if '.mlp.' in m else None
            if mlp is not None:
                # backward GEMMs: fc1 dX [M, 800] (768 real columns), fc2 dX [M, 3200] = the widths of the packs below
                bd = torch.zeros(16, N, device=self.dev, dtype=BF16)
                bu = torch.zeros(Cp if mlp == 'fc1' else self.Ip, 4, device=self.dev)
                keep += [bd, bu]
                self.wb[f'{self.pre}encoder.layers.{i}.{mlp}'] = {'lora_down': bd, 'lora_up': bu, 'lora_seg': bu.shape[0]}
                rows.append([D.data_ptr(), U.data_ptr(), K, N, ent[mlp]['lora_down'].data_ptr(),
                             ent[mlp]['lora_up'].data_ptr(), bd.data_ptr(), bu.data_ptr()])
                continue
            if is_out:
                fdown = ent['out']['lora_down'].data_ptr()
                fup = ent['out']['lora_up'].data_ptr()
            else:
                s_ = PROJ.index(m.rsplit('.', 1)[1])
                fdown = ent['qkv']['lora_down'].data_ptr() + 4 * s_ * K * 2
                fup = ent['qkv']['lora_up'].data_ptr() + s_ * Ca * 4 * 4
            # backward GEMM dX = dY W (+ alpha (dY U) D): "down" rows = U^T [16, N], "up" = alpha D^T [K (padded), 4]
            n_out = Cp if not is_out else Ca
            bd = torch.zeros(16, N, device=self.dev, dtype=BF16)
            bu = torch.zeros(n_out, 4, device=self.dev)
            keep += [bd, bu]
            self.wb[m] = {'lora_down': bd, 'lora_up': bu, 'lora_seg': n_out}
            rows.append([D.data_ptr(), U.data_ptr(), K, N, fdown, fup, bd.data_ptr(), bu.data_ptr()])
        self._lora_end = off
        self._keep = keep
        self.lora_table = torch.tensor(rows, dtype=torch.int64, device=self.dev)
        if lora is not None:
            self.load_lora_state_dict(lora)

    def load_lora_state_dict(self, lora):
        """reference checkpoint tensors ([r, 768] / [768, r], trainer_edlora.py:371-378) -> padded flat layout."""
        for m, (D, U, _, _, K, N) in self.lora_views.items():
            d = lora[f'{m}.lora_down.weight'].detach().to(self.dev, F32)
            u = lora[f'{m}.lora_up.weight'].detach().to(self.dev, F32)
            d, u = d.reshape(d.shape[0], -1), u.reshape(u.shape[0], -1)
            D.zero_()
            U.zero_()
            if m.endswith('fc1'):
                D[:d.shape[0]] = d
                U[:self.I, :u.shape[1]] = u
            elif m.endswith('fc2'):
                D[:d.shape[0], :self.I] = d
                U[:, :u.shape[1]] = u
            elif m.endswith('out_proj'):
                D[:d.shape[0]] = self._pad_heads_cols(d)
                U[:, :u.shape[1]] = u
            else:
                D[:d.shape[0]] = d
                U[:, :u.shape[1]] = self._pad_heads_rows(u)
        self.refresh_lora()

    def _unpad(self, m, D, U):
        if m.endswith('fc1'):
            return D, U[:self.I]
        if m.endswith('fc2'):
            return D[:, :self.I], U
        if m.endswith('out_proj'):
            return D.view(4, self.heads, self.dh)[:, :, :self.d].reshape(4, self.C), U
        return D, U.view(self.heads, self.dh, 4)[:, :self.d].reshape(self.C, 4)

    def lora_state_dict(self):
        out = {}
        for m, (D, U, _, _, _, _) in self.lora_views.items():
            d, u = self._unpad(m, D, U)
            out[f'{m}.lora_down.weight'] = d.clone()
            out[f'{m}.lora_up.weight'] = u.clone()
        return out

    def lora_grad_dict(self):
        out = {}
        for m, (_, _, gD, gU, _, _) in self.lora_views.items():
            d, u = self._unpad(m, gD, gU)
            out[m] = (d.clone(), u.clone())
        return out

    def refresh_lora(self):
        """Re-pack the flat LoRA parameters into the forward / backward GEMM operand layouts and write the trained embedding
        rows back into the token table (after load / optimiser step); a frozen group issues nothing."""
        if self.lora_views:
            ops.lora_pack(self.lora_table, self.lora_table.shape[0], self.alpha)
        if self.train_rows:
            self.tok.index_copy_(0, self.rows_dev.long(), self.emb_view)

    # ------------------------------------------------------------------------------------------ backward packs
    def _build_backward_packs(self):
        C, Cp, Ca = self.C, self.Cp, self.Ca
        for i in range(self.n_layers):
            ent = self.w[i]
            L = f'{self.pre}encoder.layers.{i}.'
            Wqkv = ent['qkv']['W']                                   # [3*Ca, C]
            for s_, pj in enumerate(PROJ[:3]):
                Wt = torch.zeros(Cp, Ca, device=self.dev, dtype=BF16)
                Wt[:C] = Wqkv[s_ * Ca:(s_ + 1) * Ca].t()
                self.wb.setdefault(L + 'self_attn.' + pj, {}).update(W=Wt.contiguous(), bias=None, N=Cp, K=Ca)
            Wo = ent['out']['W']                                     # [Cp, Ca]
            self.wb.setdefault(L + 'self_attn.out_proj', {}).update(W=Wo[:C].t().contiguous(), bias=None, N=Ca, K=C)
            W1 = ent['fc1']['W']                                     # [Ip, C]
            Wt = torch.zeros(Cp, self.Ip, device=self.dev, dtype=BF16)
            Wt[:C] = W1.t()
            self.wb.setdefault(L + 'fc1', {}).update(W=Wt.contiguous(), bias=None)
            W2 = ent['fc2']['W']                                     # [Cp, Ip]
            self.wb.setdefault(L + 'fc2', {}).update(W=W2[:C].t().contiguous(), bias=None)        # [Ip, C]

    def _gemm_b(self, A, ent, out, *, M, residual=None, heads=None, lda=None):
        kw = {}
        if 'lora_down' in ent:
            kw = dict(lora_down=ent['lora_down'], lora_up=ent['lora_up'], lora_seg=ent['lora_seg'])
        ops.gemm(A, ent['W'], out, M=M, residual=residual, heads=heads, lda=lda, **kw)
        self.launches += 1

    def _lg_ws(self, K, N):
        need = 128 * 4 * (K + N)
        cur = getattr(self, '_lg_buf', None)
        if cur is None or cur.numel() < need:
            self._lg_buf = torch.empty(max(need, 1 << 18), device=self.dev)
        return self._lg_buf

    def _lora_grad(self, m, x, dy, M, ldx=None, lddy=None):
        if not self.lora_views:
            return                  # frozen text encoder: no LoRA gradient
        D, U, gD, gU, K, N = self.lora_views[m]
        ops.lora_grad(x, dy, D, U, self.alpha, self._lg_ws(K, N), gD, gU, M=M, K=K, N=N, ldx=ldx, lddy=lddy,
                      accumulate=self._accumulate)

    # ------------------------------------------------------------------------------------------ forward (training)
    def tb(self, tag, shape, dtype=BF16, zero=False):
        return self.buf('T.' + tag, shape, dtype, zero)

    def forward_train(self, input_ids=None, out=None):
        """Writes the last hidden state as bf16 [n_seq * 77, 768] into `out` (e.g. the UNet engine's in_ehs) and keeps
        what the backward needs.  With input_ids=None the ids set by `set_ids` are used and the call only enqueues kernels
        (it can be captured in a CUDA graph)."""
        n, T, C, Cp, Ca, Hh, dh = self.n_seq, self.T, self.C, self.Cp, self.Ca, self.heads, self.dh
        if input_ids is not None:
            self.set_ids(input_ids)
        M = n * T
        BH = n * Hh
        dp = _r(dh, 64)
        self.launches = 0
        ids = self.buf('ids', (M,), torch.int32)
        x = self.tb('x.0', (M, Cp), zero=True)
        ops.clip_embed(ids, self.tok, self.pos, x, T=T, C=C)
        self.saved = []
        for i in range(self.n_layers):
            ent = self.w[i]
            S = {}
            ln1 = self.tb(f'ln1.{i}', (M, C))
            ops.layernorm(x, ent['ln1'][0], ent['ln1'][1], ln1, M=M, C=C, eps=self.eps, ldx=Cp, ldy=C)
            Q = self.tb(f'Q.{i}', (BH, T, dp), zero=True)
            K = self.tb(f'K.{i}', (BH, T, dp), zero=True)
            V = self.tb(f'V.{i}', (BH, T, dp), zero=True)
            hseg = dict(seg_ptr=[Q, K, V], seg_kind=[MOS_SEG_ROWS] * 3, seg_rows_pad=[T, T, T], heads=Hh, head_dim=dh,
                        dpad=dp, dv_pad=dh, tokens_per_batch=T)
            self._gemm(ln1, ent['qkv'], None, M=M, heads=hseg)
            Vt = self.buf('Vt', (BH, dh, _r(T, 8)), zero=True)
            ops.heads_transpose(V, Vt)
            ao = self.tb(f'ao.{i}', (M, Ca))
            lse = self.tb(f'lse.{i}', (BH, T), F32)
            ops.attention_causal(Q, K, Vt, ao.view(n, T, Ca), batch=n, heads=Hh, head_dim=dh, n=T, scale=self.d ** -0.5,
                                 lse2=lse)
            x1 = self.tb(f'x1.{i}', (M, Cp), zero=True)
            self._gemm(ao, ent['out'], x1, M=M, residual=x)
            ln2 = self.tb(f'ln2.{i}', (M, C))
            ops.layernorm(x1, ent['ln2'][0], ent['ln2'][1], ln2, M=M, C=C, eps=self.eps, ldx=Cp, ldy=C)
            hpre = self.tb(f'hpre.{i}', (M, self.Ip))
            self._gemm(ln2, ent['fc1'], hpre, M=M)
            h = self.buf('h', (M, self.Ip))
            ops.quick_gelu_fwd(hpre, h, M=M, C=self.Ip)
            x2 = self.tb(f'x.{i + 1}', (M, Cp), zero=True)
            self._gemm(h, ent['fc2'], x2, M=M, residual=x1)
            S.update(x=x, ln1=ln1, Q=Q, K=K, V=V, ao=ao, lse=lse, x1=x1, ln2=ln2, hpre=hpre)
            self.saved.append(S)
            x = x2
            self.launches += 6
        self.x_final = x
        y = out if out is not None else self.tb('y', (M, C))
        ops.layernorm(x, self.final_ln[0], self.final_ln[1], y, M=M, C=C, eps=self.eps, ldx=Cp, ldy=y.stride(0))
        self.launches += 2
        return y

    # ------------------------------------------------------------------------------------------ backward
    def backward(self, d_y, accumulate=False):
        """d_y: bf16 [n_seq * 77, ld >= 768] = d loss / d last_hidden_state (layer-major sequence order).  Accumulates the
        embedding-row and LoRA gradients into the flat state (`accumulate`: add to what is there).  Returns d(embedding
        output) [M, 800], or None with constant concept rows (the gradient of layer 0's input is then not formed)."""
        n, T, C, Cp, Ca, Hh, dh = self.n_seq, self.T, self.C, self.Cp, self.Ca, self.heads, self.dh
        M = n * T
        BH = n * Hh
        dp = _r(dh, 64)
        self._accumulate = bool(accumulate)
        d_x = self.buf('g_x_a', (M, Cp), zero=True)
        ops.layernorm_bwd(self.x_final, d_y, self.final_ln[0], d_x, M=M, C=C, eps=self.eps, ldx=Cp, lddy=d_y.stride(0),
                          lddx=Cp)
        other = self.buf('g_x_b', (M, Cp), zero=True)
        for i in reversed(range(self.n_layers)):
            S = self.saved[i]
            ent = self.w[i]
            L = f'{self.pre}encoder.layers.{i}.'
            # ---- MLP: x2 = x1 + fc2(quick_gelu(fc1(LN2(x1))))
            mlp_lora = self.where == 'CLIPEncoderLayer' and bool(self.lora_views)
            if mlp_lora:        # fc2's input, quick_gelu(hpre), is recomputed instead of kept
                h = self.buf('h', (M, self.Ip))
                ops.quick_gelu_fwd(S['hpre'], h, M=M, C=self.Ip)
                self._lora_grad(L + 'mlp.fc2', h, d_x, M, lddy=Cp)
            d_h = self.buf('g_h', (M, self.Ip))
            self._gemm_b(d_x, self.wb[L + 'fc2'], d_h, M=M, lda=Cp)                 # reduction over the 768 real columns
            d_hpre = self.buf('g_hpre', (M, self.Ip))
            ops.quick_gelu_bwd(S['hpre'], d_h, d_hpre, M=M, C=self.Ip)
            if mlp_lora:
                self._lora_grad(L + 'mlp.fc1', S['ln2'], d_hpre, M)
            d_ln = self.buf('g_ln', (M, Cp))
            self._gemm_b(d_hpre, self.wb[L + 'fc1'], d_ln, M=M)
            d_x1 = other
            ops.layernorm_bwd(S['x1'], d_ln, ent['ln2'][0], d_x1, M=M, C=C, eps=self.eps, add=d_x, ldx=Cp, lddy=Cp,
                              lddx=Cp, ldadd=Cp)
            # ---- attention: x1 = x + out_proj(attn(q, k, v)),  q|k|v = qkv(LN1(x))
            mo = L + 'self_attn.out_proj'
            self._lora_grad(mo, S['ao'], d_x1, M, lddy=Cp)
            dO = self.buf('g_dO', (BH, T, dp), zero=True)
            hs = dict(seg_ptr=[dO], seg_kind=[MOS_SEG_ROWS], seg_rows_pad=[T], heads=Hh, head_dim=dh, dpad=dp, dv_pad=dh,
                      tokens_per_batch=T)
            self._gemm_b(d_x1, self.wb[mo], None, M=M, heads=hs, lda=Cp)
            Qt = self.buf('g_Qt', (BH, dh, _r(T, 8)), zero=True)
            Kt = self.buf('g_Kt', (BH, dh, _r(T, 8)), zero=True)
            dOt = self.buf('g_dOt', (BH, dh, _r(T, 8)), zero=True)
            ops.heads_transpose(S['Q'], Qt)
            ops.heads_transpose(S['K'], Kt)
            ops.heads_transpose(dO, dOt)
            delta = self.buf('g_delta', (BH, T), F32)
            ops.attn_delta(dO, S['ao'], delta, batch=n, heads=Hh, head_dim=dh, N=T, ldo=Ca)
            dqkv = self.buf('g_dqkv', (M, 3 * Ca))
            ops.attention_bwd(S['Q'], S['K'], S['V'], dO, Qt, Kt, dOt, S['lse'], delta, dqkv[:, :Ca], dqkv[:, Ca:2 * Ca],
                              dqkv[:, 2 * Ca:], batch=n, heads=Hh, head_dim=dh, nq=T, nk=T, scale=self.d ** -0.5,
                              lddq=3 * Ca, lddk=3 * Ca, lddv=3 * Ca, causal=True)
            # d(input of layer 0) only feeds the embedding-row gradient: with constant rows it is not formed
            need_dx = i > 0 or self.train_rows
            for s_, pj in enumerate(PROJ[:3]):
                mm = L + 'self_attn.' + pj
                sl = dqkv[:, s_ * Ca:(s_ + 1) * Ca]
                self._lora_grad(mm, S['ln1'], sl, M, lddy=3 * Ca)
                if need_dx:
                    self._gemm_b(sl, self.wb[mm], d_ln, M=M, lda=3 * Ca, residual=d_ln if s_ > 0 else None)
            if need_dx:
                ops.layernorm_bwd(S['x'], d_ln, ent['ln1'][0], d_x, M=M, C=C, eps=self.eps, add=d_x1, ldx=Cp, lddy=Cp,
                                  lddx=Cp, ldadd=Cp)
            self.launches += 20
        if not self.train_rows:
            return None
        ops.clip_embed_bwd(self.buf('ids', (M,), torch.int32), d_x, self.rows_dev, self.emb_grad, C=C,
                           accumulate=self._accumulate)
        return d_x
