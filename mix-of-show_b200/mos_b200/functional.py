"""Operator-level entry points used by the drop-in `mixofshow.models.edlora` surface: each call packs the weights of
the module it is given (cached on the module, re-packed when a parameter changes) and runs the CUDA kernels.

No torch arithmetic fallback: unsupported shapes raise ValueError (mirrors the reference's fail-fast asserts).
"""
import torch

from . import ops
from ._lib import MOS_SEG_ROWS, MOS_SEG_TRANSPOSED

ACT = torch.float16        # operand type of the (inference-only) operator path, weights and activations: mos_b200/engine.py


def _r(x, m):
    return (x + m - 1) // m * m


def _version(*tensors):
    return tuple((t.data_ptr(), t._version) for t in tensors if t is not None)


def _lora_of(module):
    return getattr(module, '_mos_lora', None)


def pack_linears(modules, device):
    """Concatenate the weights of `modules` (nn.Linear or 1x1 nn.Conv2d) along N; include their LoRA descriptors."""
    Ws, bs, downs, ups, alphas = [], [], [], [], []
    for m in modules:
        W = m.weight.detach().to(device, torch.float32)
        Ws.append(W.reshape(W.shape[0], -1))
        bs.append(None if m.bias is None else m.bias.detach().to(device, torch.float32))
        l = _lora_of(m)
        if l is not None:
            d = l.lora_down.weight.detach().to(device, torch.float32)
            u = l.lora_up.weight.detach().to(device, torch.float32)
            downs.append(d.reshape(d.shape[0], -1))
            ups.append(u.reshape(u.shape[0], -1))
            alphas.append(float(l.alpha))
        else:
            downs.append(None)
            ups.append(None)
            alphas.append(0.0)
    W = torch.cat(Ws, 0)
    N, K = W.shape
    if N % 160 != 0 or K % 64 != 0:
        raise ValueError(f'unsupported projection shape [{N}, {K}]: the sm_90a GEMM needs N % 160 == 0 and K % 64 == 0')
    ent = {'N': N, 'K': K, 'W': W.to(ACT).contiguous(), 'bias': None}
    if any(b is not None for b in bs):
        ent['bias'] = torch.cat([b if b is not None else torch.zeros(w.shape[0], device=device)
                                 for b, w in zip(bs, Ws)]).contiguous()
    if any(d is not None for d in downs):
        down16 = torch.zeros(16, K, device=device)
        up = torch.zeros(N, 4, device=device)
        off = 0
        for s, (d, u, a, w) in enumerate(zip(downs, ups, alphas, Ws)):
            if d is not None:
                r = d.shape[0]
                if r > 4:
                    raise ValueError('LoRA rank > 4 is not supported by the fused epilogue')
                down16[4 * s:4 * s + r] = d
                up[off:off + w.shape[0], :r] = u * a
            off += w.shape[0]
        ent['lora_down'] = down16.to(ACT).contiguous()
        ent['lora_up'] = up.contiguous()
        ent['lora_seg'] = Ws[0].shape[0] if len(modules) > 1 else N
    return ent


def _cached(owner, key, modules, device):
    tens = []
    for m in modules:
        tens += [m.weight, m.bias]
        l = _lora_of(m)
        if l is not None:
            tens += [l.lora_down.weight, l.lora_up.weight, l.alpha]
    ver = (_version(*tens), str(device))
    cache = owner.__dict__.setdefault('_mos_pack', {})
    if key not in cache or cache[key][0] != ver:
        cache[key] = (ver, pack_linears(modules, device))
    return cache[key][1]


def _lora_kw(ent):
    if 'lora_down' in ent:
        return dict(lora_down=ent['lora_down'], lora_up=ent['lora_up'], lora_seg=ent['lora_seg'])
    return {}


def lora_linear(module, x):
    """y = module(x) + alpha * up(down(x))  — LoRALinearLayer.forward (mixofshow/models/edlora.py:244-246) as one
    fused wgmma GEMM.  module: nn.Linear or 1x1 nn.Conv2d carrying a `_mos_lora` descriptor (or none)."""
    if not x.is_cuda:
        raise ValueError('the GPU path needs CUDA tensors (there is no CPU fallback)')
    ent = _cached(module, 'self', [module], x.device)
    conv = module.__class__.__name__ == 'Conv2d'
    if conv:
        b, c, h, w = x.shape
        A = x.permute(0, 2, 3, 1).reshape(b * h * w, c).to(ACT).contiguous()
    else:
        A = x.reshape(-1, x.shape[-1]).to(ACT).contiguous()
    out = torch.empty(A.shape[0], ent['N'], device=x.device, dtype=ACT)
    ops.gemm(A, ent['W'], out, bias=ent['bias'], **_lora_kw(ent))
    if conv:
        return out.view(b, h, w, ent['N']).permute(0, 3, 1, 2).to(x.dtype)
    return out.view(*x.shape[:-1], ent['N']).to(x.dtype)


def attention_block(attn, hidden_states, encoder_hidden_states=None, want_probs=False, regions=None,
                    region_hw=None):
    """q/k/v projections (+LoRA) -> flash attention -> out projection (+LoRA, +bias) on the CUDA path.

    attn: an `Attention`-like module exposing to_q / to_k / to_v / to_out[0] (nn.Linear) and .heads.
    hidden_states [B, N, C]; encoder_hidden_states None (self) or [B, M, Cc].  regions: list of
    (region_embeds [B, M, Cc], (sh, sw, eh, ew) feature-pixel ints) for the regional rewrite.
    Returns (out [B, N, C] in hidden_states.dtype, probs fp32 [B*heads, N, M] or None)."""
    if not hidden_states.is_cuda:
        raise ValueError('the GPU path needs CUDA tensors (there is no CPU fallback)')
    dev = hidden_states.device
    B, N, C = hidden_states.shape
    Hh = attn.heads
    d = attn.to_q.weight.shape[0] // Hh
    if d not in (40, 80, 160):
        raise ValueError(f'head_dim {d} unsupported (SD1.5 uses 40 / 80 / 160)')
    inner = Hh * d
    BH = B * Hh
    dp, dv = _r(d, 64), _r(d, 16)
    x = hidden_states.reshape(B * N, C).to(ACT).contiguous()
    Q = torch.zeros(BH, N, dp, device=dev, dtype=ACT)
    if encoder_hidden_states is None:
        M = N
        ent = _cached(attn, 'qkv', [attn.to_q, attn.to_k, attn.to_v], dev)
        K = torch.zeros(BH, M, dp, device=dev, dtype=ACT)
        Vt = torch.zeros(BH, dv, _r(M, 8), device=dev, dtype=ACT)
        ops.gemm(x, ent['W'], None, heads=dict(
            seg_ptr=[Q, K, Vt], seg_kind=[MOS_SEG_ROWS, MOS_SEG_ROWS, MOS_SEG_TRANSPOSED],
            seg_rows_pad=[N, M, _r(M, 8)], heads=Hh, head_dim=d, dpad=dp, dv_pad=dv, tokens_per_batch=N),
            **_lora_kw(ent))
    else:
        M = encoder_hidden_states.shape[1]
        entq = _cached(attn, 'q', [attn.to_q], dev)
        ops.gemm(x, entq['W'], None, heads=dict(seg_ptr=[Q], seg_kind=[MOS_SEG_ROWS], seg_rows_pad=[N], heads=Hh,
                                                head_dim=d, dpad=dp, dv_pad=dv, tokens_per_batch=N),
                 **_lora_kw(entq))
        K, Vt = _project_kv(attn, encoder_hidden_states, Hh, d, dev)
    o = torch.empty(B, N, inner, device=dev, dtype=ACT)
    probs = torch.empty(BH, N, M, device=dev, dtype=torch.float32) if want_probs else None
    if want_probs and M > 128:
        raise ValueError('attention-probability output is limited to one key tile (cross-attention, <= 128 keys)')
    ops.attention(Q, K, Vt, o, batch=B, heads=Hh, head_dim=d, nq=N, nk=M, scale=float(attn.scale), probs=probs)
    if regions:
        fh, fw = region_hw
        outs, boxes = [], []
        for emb, box in regions:
            Kr, Vr = _project_kv(attn, emb, Hh, d, dev)
            orr = torch.empty_like(o)
            ops.attention(Q, Kr, Vr, orr, batch=B, heads=Hh, head_dim=d, nq=N, nk=emb.shape[1],
                          scale=float(attn.scale))
            outs.append(orr)
            boxes.append(box)
        ptrs = torch.tensor([t.data_ptr() for t in outs], dtype=torch.int64, device=dev)
        ops.region_combine(o, ptrs, boxes, o, B=B, FH=fh, FW=fw, C=inner, ld=inner)
    ento = _cached(attn, 'out', [attn.to_out[0]], dev)
    y = torch.empty(B * N, ento['N'], device=dev, dtype=ACT)
    ops.gemm(o.view(B * N, inner), ento['W'], y, bias=ento['bias'], **_lora_kw(ento))
    return y.view(B, N, -1).to(hidden_states.dtype), probs


def _project_kv(attn, ehs, Hh, d, dev):
    B, M, Cc = ehs.shape
    dp, dv = _r(d, 64), _r(d, 16)
    ent = _cached(attn, 'kv', [attn.to_k, attn.to_v], dev)
    e = ehs.reshape(B * M, Cc).to(ACT).contiguous()
    K = torch.zeros(B * Hh, M, dp, device=dev, dtype=ACT)
    Vt = torch.zeros(B * Hh, dv, _r(M, 8), device=dev, dtype=ACT)
    ops.gemm(e, ent['W'], None, heads=dict(seg_ptr=[K, Vt], seg_kind=[MOS_SEG_ROWS, MOS_SEG_TRANSPOSED],
                                           seg_rows_pad=[M, _r(M, 8)], heads=Hh, head_dim=d, dpad=dp, dv_pad=dv,
                                           tokens_per_batch=M), **_lora_kw(ent))
    return K, Vt
