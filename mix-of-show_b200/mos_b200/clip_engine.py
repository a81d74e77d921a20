"""CLIPTextEngine — the CLIP text encoder forward on the GPU (SURVEY.md §8f rank 1), built only from libmos_sm100 kernels.

Owns the `text_encoder(input_ids)[0]` call the reference makes at mixofshow/pipelines/pipeline_edlora.py:133-145,
trainer_edlora.py:220-234 and gradient_fusion.py:182-199 (transformers `CLIPTextModel`: token + position embeddings,
12 pre-LN layers of causal self-attention and a quick-GELU MLP, final LayerNorm), with the ED-LoRA of `where: CLIPAttention`
(q_proj / k_proj / v_proj / out_proj, trainer_edlora.py:107-118) fused into the projection GEMMs exactly as in the UNet;
with `where: CLIPEncoderLayer` the LoRA of mlp.fc1 / mlp.fc2 is fused into the MLP GEMMs the same way.

Shapes are bent to the GEMM kernel's 160-column tiles without touching the arithmetic:
  * hidden states live in [M, 800] buffers (768 real columns, the rest stays zero: zero weight rows / bias);
  * the 12 heads of 64 dims run as head_dim 80 (16 zero columns per head in q, k, v; `scale` stays 64^-0.5), so the fused
    q|k|v projection has N = 3 * 12 * 80 = 2880 = 18 tiles and feeds the existing head-split epilogue and the d = 80
    attention kernel (causal variant); out_proj reads K = 960 with zero weight columns at the pads;
  * fc1 is padded 3072 -> 3200 (quick-GELU(0) = 0), fc2 reads K = 3200; their LoRA up rows / down columns are padded
    the same way with zeros.
There is no CPU / PyTorch fallback: every arithmetic op is a C-ABI call.
"""
import torch

from . import ops
from ._lib import MOS_SEG_ROWS, MOS_SEG_TRANSPOSED

BF16 = torch.bfloat16
PROJ = ('q_proj', 'k_proj', 'v_proj', 'out_proj')


def _r(x, m):
    return (x + m - 1) // m * m


class CLIPTextEngine:
    def __init__(self, state_dict, n_seq, *, lora=None, lora_alpha=1.0, merge_lora=False, device='cuda', heads=12,
                 prefix='text_model.', eps=1e-5):
        """state_dict: transformers CLIPTextModel parameter names (fp32).  lora: {f'{module}.lora_down.weight' [r, 768],
        f'{module}.lora_up.weight' [768, r]} with module = 'text_model.encoder.layers.{i}.self_attn.{q,k,v,out}_proj'
        and optionally 'text_model.encoder.layers.{i}.mlp.fc{1,2}' ([r, 768] / [3072, r] and [r, 3072] / [768, r])
        (EDLoRATrainer.delta_state_dict()['text_encoder'], trainer_edlora.py:371-378); rank <= 4.
        n_seq: number of 77-token sequences per call (16 per prompt for the layer-wise embeddings)."""
        self.dev = torch.device(device)
        self.pre = prefix
        sd = state_dict
        self.C = sd[prefix + 'embeddings.token_embedding.weight'].shape[1]
        self.T = sd[prefix + 'embeddings.position_embedding.weight'].shape[0]
        self.heads = heads
        self.d = self.C // heads                     # 64
        self.dh = 80                                 # head_dim the (causal) attention kernel runs; heads are zero padded
        assert self.d <= self.dh, f'head dim {self.d} > 80 is not supported'
        self.Cp = _r(self.C, 160)                    # 800
        self.Ca = heads * self.dh                    # 960: attention output width (padded heads)
        self.n_seq = n_seq
        self.eps = eps
        self.lora = None if merge_lora else lora
        self._merge = lora if merge_lora else None
        self.alpha = float(lora_alpha)
        self.n_layers = 1 + max(int(k.split('.layers.')[1].split('.')[0]) for k in sd if '.layers.' in k)
        self.I = sd[f'{prefix}encoder.layers.0.mlp.fc1.weight'].shape[0]
        self.Ip = _r(self.I, 160)                    # 3200
        self.w = {}
        self.bufs = {}
        self.gram_rec = None        # gradient fusion: callable(key, A [M, C] bf16 view, M, C)
        self.launches = 0
        f32 = lambda k: sd[k].detach().to(self.dev, torch.float32)
        self.tok = f32(prefix + 'embeddings.token_embedding.weight').contiguous()
        self.pos = f32(prefix + 'embeddings.position_embedding.weight').contiguous()
        self.final_ln = (f32(prefix + 'final_layer_norm.weight').contiguous(), f32(prefix + 'final_layer_norm.bias').contiguous())
        for i in range(self.n_layers):
            self._pack_layer(i, f32)

    def set_token_embedding(self, table):
        """Re-upload the token-embedding table (new concept rows written by the caller, trainer_edlora.py:77-82 /
        convert_edlora_to_diffusers.py:17-20); the row count may have grown (resize_token_embeddings)."""
        self.tok = table.detach().to(self.dev, torch.float32).contiguous()

    # ------------------------------------------------------------------------------------------ packing
    def _lora_pair(self, module):
        src = self._merge if self._merge is not None else self.lora
        if src is None or f'{module}.lora_down.weight' not in src:
            return None
        d = src[f'{module}.lora_down.weight'].detach().to(self.dev, torch.float32)
        u = src[f'{module}.lora_up.weight'].detach().to(self.dev, torch.float32)
        return d.reshape(d.shape[0], -1), u.reshape(u.shape[0], -1)

    def _head_rows(self, W):
        """[heads*d, K] -> [heads*dh, K]: every head's d rows followed by dh - d zero rows."""
        K = W.shape[1]
        out = torch.zeros(self.heads, self.dh, K, device=self.dev)
        out[:, :self.d] = W.reshape(self.heads, self.d, K)
        return out.reshape(self.heads * self.dh, K)

    def _pack_layer(self, i, f32):
        L = f'{self.pre}encoder.layers.{i}.'
        C, Cp, Ca = self.C, self.Cp, self.Ca
        ent = {}
        ent['ln1'] = (f32(L + 'layer_norm1.weight').contiguous(), f32(L + 'layer_norm1.bias').contiguous())
        ent['ln2'] = (f32(L + 'layer_norm2.weight').contiguous(), f32(L + 'layer_norm2.bias').contiguous())
        # ---- fused q|k|v: N = 3 * heads * dh, rows padded per head
        Ws, bs, down16, up = [], [], torch.zeros(16, C, device=self.dev), torch.zeros(3 * Ca, 4, device=self.dev)
        any_lora = False
        for s_, pj in enumerate(PROJ[:3]):
            m = L + 'self_attn.' + pj
            W, b = f32(m + '.weight'), f32(m + '.bias')
            pair = self._lora_pair(m)
            if pair is not None and self._merge is not None:
                W = W + self.alpha * (pair[1] @ pair[0])          # merge_lora_into_weight, gradient_fusion.py:99-143
                pair = None
            Ws.append(self._head_rows(W))
            bs.append(self._head_rows(b[:, None])[:, 0])
            if pair is not None:
                any_lora = True
                r = pair[0].shape[0]
                assert r <= 4, 'LoRA rank > 4 is not supported by the fused epilogue'
                down16[4 * s_:4 * s_ + r] = pair[0]
                up[s_ * Ca:(s_ + 1) * Ca, :r] = self._head_rows(pair[1]) * self.alpha
        ent['qkv'] = {'W': torch.cat(Ws, 0).to(BF16).contiguous(), 'bias': torch.cat(bs, 0).contiguous()}
        if any_lora:
            ent['qkv'].update(lora_down=down16.to(BF16).contiguous(), lora_up=up.contiguous(), lora_seg=Ca)
        # ---- out_proj: N padded 768 -> 800 (zero rows), K = heads * dh (zero columns at the head pads)
        m = L + 'self_attn.out_proj'
        W, b = f32(m + '.weight'), f32(m + '.bias')
        pair = self._lora_pair(m)
        if pair is not None and self._merge is not None:
            W = W + self.alpha * (pair[1] @ pair[0])
            pair = None

        def pad_k(Wk):          # [n, heads*d] -> [n, heads*dh]
            n = Wk.shape[0]
            out = torch.zeros(n, self.heads, self.dh, device=self.dev)
            out[:, :, :self.d] = Wk.reshape(n, self.heads, self.d)
            return out.reshape(n, Ca)

        Wp = torch.zeros(Cp, Ca, device=self.dev)
        Wp[:C] = pad_k(W)
        bp = torch.zeros(Cp, device=self.dev)
        bp[:C] = b
        ent['out'] = {'W': Wp.to(BF16).contiguous(), 'bias': bp.contiguous()}
        if pair is not None:
            r = pair[0].shape[0]
            d16 = torch.zeros(16, Ca, device=self.dev)
            d16[:r] = pad_k(pair[0])
            u4 = torch.zeros(Cp, 4, device=self.dev)
            u4[:C, :r] = pair[1] * self.alpha
            ent['out'].update(lora_down=d16.to(BF16).contiguous(), lora_up=u4.contiguous(), lora_seg=Cp)
        # ---- MLP: fc1 N padded to Ip, fc2 K = Ip, N padded to Cp
        W1 = torch.zeros(self.Ip, C, device=self.dev)
        W1[:self.I] = self._mlp_weight(L + 'mlp.fc1', f32)
        b1 = torch.zeros(self.Ip, device=self.dev)
        b1[:self.I] = f32(L + 'mlp.fc1.bias')
        ent['fc1'] = {'W': W1.to(BF16).contiguous(), 'bias': b1.contiguous()}
        W2 = torch.zeros(Cp, self.Ip, device=self.dev)
        W2[:C, :self.I] = self._mlp_weight(L + 'mlp.fc2', f32)
        b2 = torch.zeros(Cp, device=self.dev)
        b2[:C] = f32(L + 'mlp.fc2.bias')
        ent['fc2'] = {'W': W2.to(BF16).contiguous(), 'bias': b2.contiguous()}
        pair = self._lora_pair(L + 'mlp.fc1') if self._merge is None else None
        if pair is not None:                 # down [r, 768] as is, up rows padded 3072 -> 3200
            r = pair[0].shape[0]
            assert r <= 4, 'LoRA rank > 4 is not supported by the fused epilogue'
            d16 = torch.zeros(16, C, device=self.dev)
            d16[:r] = pair[0]
            u4 = torch.zeros(self.Ip, 4, device=self.dev)
            u4[:self.I, :r] = pair[1] * self.alpha
            ent['fc1'].update(lora_down=d16.to(BF16).contiguous(), lora_up=u4.contiguous(), lora_seg=self.Ip)
        pair = self._lora_pair(L + 'mlp.fc2') if self._merge is None else None
        if pair is not None:                 # down columns padded 3072 -> 3200, up rows 768 -> 800
            r = pair[0].shape[0]
            assert r <= 4, 'LoRA rank > 4 is not supported by the fused epilogue'
            d16 = torch.zeros(16, self.Ip, device=self.dev)
            d16[:r, :self.I] = pair[0]
            u4 = torch.zeros(Cp, 4, device=self.dev)
            u4[:C, :r] = pair[1] * self.alpha
            ent['fc2'].update(lora_down=d16.to(BF16).contiguous(), lora_up=u4.contiguous(), lora_seg=Cp)
        self.w[i] = ent

    def _mlp_weight(self, m, f32):
        """fc1 / fc2 weight, with a merged LoRA folded in (merge_lora_into_weight, gradient_fusion.py:99-143)"""
        W = f32(m + '.weight')
        if self._merge is not None:
            pair = self._lora_pair(m)
            if pair is not None:
                W = W + self.alpha * (pair[1] @ pair[0])
        return W

    # ------------------------------------------------------------------------------------------ forward
    def buf(self, name, shape, dtype=BF16, zero=False):
        key = (name, tuple(shape), dtype)
        if key not in self.bufs:
            self.bufs[key] = (torch.zeros if zero else torch.empty)(shape, device=self.dev, dtype=dtype)
        return self.bufs[key]

    def _gemm(self, A, ent, out, *, M, residual=None, heads=None, lda=None):
        kw = {}
        if 'lora_down' in ent:
            kw = dict(lora_down=ent['lora_down'], lora_up=ent['lora_up'], lora_seg=ent['lora_seg'])
        ops.gemm(A, ent['W'], out, M=M, bias=ent['bias'], residual=residual, heads=heads, lda=lda, **kw)
        self.launches += 1

    def set_ids(self, input_ids):
        """input_ids: integer [n_seq, 77] -> the static id buffer `encode` (and the training engine's forward / backward)
        reads, so that those calls only enqueue kernels and can be captured in a CUDA graph."""
        assert tuple(input_ids.shape) == (self.n_seq, self.T), \
            f'expected ids of shape {(self.n_seq, self.T)}, got {tuple(input_ids.shape)}'
        self.buf('ids', (self.n_seq * self.T,), torch.int32).copy_(input_ids.reshape(-1).to(self.dev, torch.int32))

    def forward(self, input_ids):
        """input_ids: integer tensor [n_seq, 77] -> last_hidden_state fp32 [n_seq, 77, 768] (after final_layer_norm)."""
        self.set_ids(input_ids)
        y = self.encode(self.buf('y', (self.n_seq * self.T, self.C)))
        return y.float().view(self.n_seq, self.T, self.C)

    def encode(self, out):
        """last_hidden_state of the ids set by `set_ids` as bf16 rows [n_seq * 77, 768] of pitch out.stride(0) (e.g. a
        training engine's in_ehs); saves nothing for a backward pass and only enqueues kernels."""
        n, T, C, Cp, Ca, Hh, dh = self.n_seq, self.T, self.C, self.Cp, self.Ca, self.heads, self.dh
        M = n * T
        self.launches = 0
        ids = self.buf('ids', (M,), torch.int32)
        x = self.buf('x0', (M, Cp))
        ops.clip_embed(ids, self.tok, self.pos, x, T=T, C=C)
        self.launches += 1
        ln = self.buf('ln', (M, C))
        BH = n * Hh
        Q = self.buf('Q', (BH, T, _r(dh, 64)), zero=True)
        K = self.buf('K', (BH, T, _r(dh, 64)), zero=True)
        Vt = self.buf('Vt', (BH, dh, _r(T, 8)), zero=True)
        ao = self.buf('ao', (M, Ca))
        hseg = dict(seg_ptr=[Q, K, Vt], seg_kind=[MOS_SEG_ROWS, MOS_SEG_ROWS, MOS_SEG_TRANSPOSED],
                    seg_rows_pad=[T, T, _r(T, 8)], heads=Hh, head_dim=dh, dpad=_r(dh, 64), dv_pad=dh, tokens_per_batch=T)
        for i in range(self.n_layers):
            ent = self.w[i]
            key = f'{self.pre}encoder.layers.{i}.'
            ops.layernorm(x, ent['ln1'][0], ent['ln1'][1], ln, M=M, C=C, eps=self.eps, ldx=Cp, ldy=C)
            if self.gram_rec is not None:
                self.gram_rec(key + 'self_attn.in', ln, M, C)
            self._gemm(ln, ent['qkv'], None, M=M, heads=hseg)
            ops.attention_causal(Q, K, Vt, ao.view(n, T, Ca), batch=n, heads=Hh, head_dim=dh, n=T, scale=self.d ** -0.5)
            if self.gram_rec is not None:
                self.gram_rec(key + 'self_attn.out_proj', ao, M, Ca)
            x1 = self.buf(f'x1_{i & 1}', (M, Cp))
            self._gemm(ao, ent['out'], x1, M=M, residual=x)
            ops.layernorm(x1, ent['ln2'][0], ent['ln2'][1], ln, M=M, C=C, eps=self.eps, ldx=Cp, ldy=C)
            if self.gram_rec is not None:
                self.gram_rec(key + 'mlp.fc1', ln, M, C)
            h = self.buf('h', (M, self.Ip))
            self._gemm(ln, ent['fc1'], h, M=M)
            ops.quick_gelu(h, M=M, C=self.Ip)
            if self.gram_rec is not None:
                self.gram_rec(key + 'mlp.fc2', h[:, :self.I], M, self.I)     # the I real columns of the padded buffer
            x2 = self.buf(f'x2_{i & 1}', (M, Cp))
            self._gemm(h, ent['fc2'], x2, M=M, residual=x1)
            x = x2
            self.launches += 4
        ops.layernorm(x, self.final_ln[0], self.final_ln[1], out, M=M, C=C, eps=self.eps, ldx=Cp, ldy=out.stride(0))
        self.launches += 1
        return out

    __call__ = forward
