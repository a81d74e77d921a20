"""Helpers shared by the kernel parity tests: seeded inputs, the rel-L2 metric, head packing and canary buffers.

A canary buffer is an output allocation larger than the kernel's logical output window, filled with a sentinel bit pattern
(a NaN in bf16, fp16 and fp32).  After the launch everything outside the window must still hold the sentinel.
"""
import torch

SENTINEL = {2: 0x7FA5, 4: 0x7FA5A5A5}          # element size -> bit pattern
_INT = {2: torch.int16, 4: torch.int32}


def rel_l2(a, b):
    a, b = a.float(), b.float()
    return ((a - b).norm() / b.norm().clamp_min(1e-12)).item()


def rel_l2_64(a, b):
    """rel_l2 evaluated in float64, for fp32 kernels against float64 references"""
    a, b = a.double(), b.double()
    return ((a - b).norm() / b.norm().clamp_min(1e-300)).item()


def mk(shape, dev, scale=1.0, seed=0, dtype=torch.bfloat16):
    g = torch.Generator(device='cpu').manual_seed(seed)
    return (torch.randn(shape, generator=g) * scale).to(dev).to(dtype)


def bits(t):
    """the raw bits of a 16- or 32-bit tensor (for bitwise comparisons that also hold for NaN patterns)"""
    return t.view(_INT[t.element_size()])


def same_bits(a, b):
    return torch.equal(bits(a), bits(b))


def canary(shape, dev, dtype):
    t = torch.empty(shape, device=dev, dtype=dtype)
    bits(t).fill_(SENTINEL[t.element_size()])
    return t


def untouched(buf, window):
    """True if every element of `buf` outside the boolean mask `window` still holds the sentinel"""
    return bool((bits(buf)[~window] == SENTINEL[buf.element_size()]).all())


def window_mask(buf, *index):
    m = torch.zeros(buf.shape, dtype=torch.bool, device=buf.device)
    m[index] = True
    return m


def num_sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def rup(x, m):
    return (x + m - 1) // m * m


def gn_path(B, HW, C, ldx, ldy, sms=None):
    """The GroupNorm forward implementation `mos_groupnorm_fwd` picks for these arguments (unless the two-pass switch is
    on): ('cluster', k, vec) for the one-pass kernel with a cluster of k CTAs and vec-element words, or 'fallback' for
    the statistics + apply launches.  A copy of the host rule in csrc/norm.cu, mos_groupnorm_fwd ("one-pass path" block:
    the vec choice, the k-widening loop and the 200 KB shared-memory test); keep the two in step."""
    import os
    sms = num_sms() if sms is None else sms
    cpg = C // 32
    vec = 4 if cpg % 4 == 0 and ldx % 4 == 0 and ldy % 4 == 0 else 2
    slab = HW * cpg * 2
    min_ctas = int(os.environ.get('MOS_GN_MIN_CTAS', '0')) or 2 * sms
    if min_ctas < 1:
        min_ctas = 2 * sms
    k = 1
    while k < 8 and HW // (2 * k) >= 16 and (slab // k > 48 * 1024 or B * 32 * k < min_ctas):
        k *= 2
    smem = -(-HW // k) * cpg * 2
    if smem <= 200 * 1024 and cpg % 2 == 0 and ldx % 2 == 0 and ldy % 2 == 0:
        return ('cluster', k, vec)
    return 'fallback'


def plant_outlier(x, C, layout, K, seed):
    """x [B, HW, ld] with NaN pad columns; returns a copy in which the group's first element of row 0 (layout 'pivot'), or
    all C channels of row 0 (layout 'corner': the top-left pixel, where the zero padding of 3x3 convolutions leaves its
    mark), lies K x the group's std away from the group's mean, with a random sign per (sample, group).  K = 'max' is
    sqrt(n) / 2 for the group size n = HW * C / 32: one element can lie at most sqrt(n - 1) std from its group's mean.
    Also returns the boolean mask of the planted elements over [B, HW, C]."""
    B, HW = x.shape[:2]
    cpg = C // 32
    if K == 'max':
        K = (HW * cpg) ** 0.5 / 2
    g = torch.Generator(device='cpu').manual_seed(seed)
    sign = torch.where(torch.rand(B, 1, 32, 1, generator=g) < 0.5, -1.0, 1.0).to(x.device)
    body = x[..., :C].double().view(B, HW, 32, cpg)
    mean = body.mean(dim=(1, 3), keepdim=True)
    std = body.std(dim=(1, 3), keepdim=True)
    mask = torch.zeros(B, HW, 32, cpg, dtype=torch.bool, device=x.device)
    if layout == 'pivot':
        mask[:, 0, :, 0] = True
    else:
        mask[:, 0] = True
    planted = torch.where(mask, mean + sign * K * std, body)
    out = x.clone()
    out[..., :C] = planted.view(B, HW, C).to(x.dtype)
    return out, mask.view(B, HW, C)


def worst_group_rel_l2(y, ref, C):
    """the largest rel-L2 over the (sample, group) pairs of [B, HW, C] outputs"""
    B, HW = y.shape[:2]
    d = (y.double() - ref.double()).view(B, HW, 32, C // 32)
    r = ref.double().view(B, HW, 32, C // 32)
    return (d.norm(dim=(1, 3)) / r.norm(dim=(1, 3)).clamp_min(1e-300)).max().item()


def pack_rows(t, dp):
    """[B, H, n, d] -> the zero-padded head-split row layout [B*H, n, dp]"""
    B, H, n, d = t.shape
    out = torch.zeros(B * H, n, dp, device=t.device, dtype=t.dtype)
    out[..., :d] = t.reshape(B * H, n, d)
    return out


def pack_vt(v, dv):
    """[B, H, nk, d] -> the zero-padded transposed layout [B*H, dv, nk rounded up to 8]"""
    B, H, nk, d = v.shape
    out = torch.zeros(B * H, dv, rup(nk, 8), device=v.device, dtype=v.dtype)
    out[:, :d, :nk] = v.reshape(B * H, nk, d).transpose(1, 2)
    return out
