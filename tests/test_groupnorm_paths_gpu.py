"""GroupNorm forward (csrc/norm.cu, mos_groupnorm_fwd) on both of its implementations.

The entry point picks the one-pass cluster kernel (a cluster of k = 1, 2, 4 or 8 CTAs keeps one (sample, group) slab in
shared memory, vec = 2 or 4 elements per word) when the slab fits 8 x 200 KB, and otherwise the two-launch fallback
(statistics kernel + apply kernel through a fp32 workspace).  The VAE at 512 x 512 takes the fallback for its
HW = 262144 layers and for C = 512 at HW = 65536; every UNet shape takes the cluster kernel.  Each case below runs on the
path the host rule picks and, through `mos_debug_set_gn_twopass`, on the forced fallback.

Reference: F.group_norm in float64 on the same rounded 16-bit input, then SiLU where asked.  Bounds are those of
test_kernels_gpu.py / test_f16_kernels_gpu.py: rel-L2 < 4e-3 for bf16 outputs and < 6e-4 for fp16 (one output rounding
plus fp32 statistics).  Offset activations (group mean up to 100 x the group's std) are held to the same bounds: PyTorch's
GroupNorm meets them at any offset the 16-bit input can represent.

Test ids carry the path that an H100 (132 SMs) takes; `test_case_list_covers_every_path` checks the coverage on the device
the suite runs on.
"""
import contextlib

import pytest
import torch
import torch.nn.functional as F

from gpu_helpers import (canary, gn_path, num_sms, plant_outlier, rel_l2, rup, same_bits, untouched, window_mask,
                         worst_group_rel_l2)

pytestmark = pytest.mark.gpu
BF, H16 = torch.bfloat16, torch.float16
TOL = {BF: 4e-3, H16: 6e-4}
H100_SMS = 132

# (name, B, HW, C, ldx, ldy, dtype, silu, eps)
VAE = [(f'vae{B}', B, HW, C, rup(C, 160), C, H16, True, 1e-6)
       for B in (1, 2)
       for C, HW in [(128, 262144), (128, 65536), (256, 262144), (256, 65536), (256, 16384), (512, 65536), (512, 16384),
                     (512, 4096)]]
VAE.append(('vae-attn', 1, 4096, 512, 640, 512, H16, False, 1e-6))     # mid-block attention norm: no SiLU
UNET = [(f'unet-{"bf16" if dt == BF else "fp16"}', B, HW, C, ld, C + 32, dt, silu, 1e-5)
        for dt in (BF, H16)
        for B, HW, C, ld, silu in [(2, 4096, 320, 320, True), (2, 1024, 640, 1280, True), (2, 256, 1280, 1280, True),
                                   (2, 256, 2560, 2560, True), (2, 64, 1280, 1280, False), (2, 64, 2560, 2560, True),
                                   (1, 4096, 960, 960, True), (2, 1024, 1920, 1920, True)]]
# small batches / maps: the cluster width k follows from B * 32 * k >= 2 x SM count and HW / (2k) >= 16
SMALL = [('k1', 9, 64, 320, 320, 320, BF, True, 1e-5), ('k1-tail', 9, 100, 960, 960, 960, H16, True, 1e-5),
         ('k1-hw16', 2, 16, 640, 640, 648, H16, False, 1e-5), ('k2', 6, 256, 640, 640, 640, BF, True, 1e-5),
         ('k2-hw32', 1, 32, 320, 320, 328, H16, True, 1e-5), ('k4', 3, 288, 320, 320, 320, BF, False, 1e-5),
         ('k4-cpg30', 4, 64, 960, 960, 968, H16, True, 1e-5), ('odd-cpg', 2, 1000, 96, 96, 104, BF, True, 1e-5)]
CASES = VAE + UNET + SMALL


def _label(case):
    name, B, HW, C, ldx, ldy = case[:6]
    p = gn_path(B, HW, C, ldx, ldy, sms=H100_SMS)
    path = 'fallback' if p == 'fallback' else f'k{p[1]}v{p[2]}'
    return f'{name}-B{B}-HW{HW}-C{C}-{path}'


@contextlib.contextmanager
def forced_fallback(on=True):
    """`mos_debug_set_gn_twopass` is a process-global switch: always put it back to the default."""
    from mos_b200 import _lib
    _lib.lib().mos_debug_set_gn_twopass(1 if on else 0)
    try:
        yield
    finally:
        _lib.lib().mos_debug_set_gn_twopass(0)


@pytest.fixture(params=['auto', 'fallback'])
def gn_mode(request, cuda):
    with forced_fallback(request.param == 'fallback'):
        yield request.param


def _expected(mode, B, HW, C, ldx, ldy):
    return 'fallback' if mode == 'fallback' else gn_path(B, HW, C, ldx, ldy)


def _input(B, HW, C, ldx, dtype, dev, ratio=0.0, seed=0, const=False):
    """x [B, HW, ldx]: group g of sample b is s * (ratio * sign + spread_c + noise) with a per-(sample, group) scale s in
    [0.5, 2] and a per-channel spread, so the group mean / std is about `ratio`; const=True drops spread and noise (every
    group is one value).  The pad columns C..ldx are NaN."""
    g = torch.Generator(device=dev).manual_seed(seed)
    cpg = C // 32
    scale = torch.exp2(torch.rand(B, 1, 32, 1, generator=g, device=dev) * 2 - 1)
    sign = torch.where(torch.rand(B, 1, 32, 1, generator=g, device=dev) < 0.5, -1.0, 1.0)
    spread = torch.randn(1, 1, 32, cpg, generator=g, device=dev) * 0.6
    noise = torch.randn(B, HW, 32, cpg, generator=g, device=dev) * 0.8
    if const:
        body = scale * (sign * (ratio + torch.arange(32, device=dev).view(1, 1, 32, 1) * 0.37)).expand(B, HW, 32, cpg)
    else:
        body = scale * (ratio * sign + spread + noise)
    x = torch.full((B, HW, ldx), float('nan'), device=dev, dtype=dtype)
    x[..., :C] = body.reshape(B, HW, C).to(dtype)
    return x


def _affine(C, dev, seed=1):
    g = torch.Generator(device=dev).manual_seed(seed)
    return torch.randn(C, generator=g, device=dev), torch.randn(C, generator=g, device=dev)


def _reference(x, C, gamma, beta, eps, silu):
    r = F.group_norm(x[..., :C].double().transpose(1, 2), 32, gamma.double(), beta.double(), eps)
    return (F.silu(r) if silu else r).transpose(1, 2)


def _run(x, gamma, beta, B, HW, C, ldy, dtype, eps, silu, partial=None):
    """y into a canary buffer [B*HW + 3, ldy]: returns (the whole buffer, the [B, HW, C] output view, the workspace).
    The default workspace is the engines' B*592*64 floats, sentinel-filled: only the fallback writes to it."""
    from mos_b200 import ops
    dev = x.device
    buf = canary((B * HW + 3, ldy), dev, dtype)
    part = canary((B * 592 * 64,), dev, torch.float32) if partial is None else partial
    ops.groupnorm(x, gamma, beta, buf, part, B=B, HW=HW, C=C, eps=eps, silu=silu, ldx=x.shape[-1], ldy=ldy)
    torch.cuda.synchronize()
    return buf, buf[:B * HW, :C].view(B, HW, C), part


def _window(buf, B, HW, C):
    return window_mask(buf, slice(0, B * HW), slice(0, C))


def test_case_list_covers_every_path(cuda):
    """The cases below reach cluster widths 1, 2, 4 and 8, vec 2 with cpg 10 and 30, vec 4, and the fallback without
    forcing, on this device."""
    paths = {gn_path(*c[1:6]) for c in CASES}
    clusters = {p for p in paths if p != 'fallback'}
    assert {p[1] for p in clusters} >= {1, 2, 4, 8}, paths
    assert 'fallback' in paths
    assert any(p[2] == 4 for p in clusters)
    vec2_cpg = {c[3] // 32 for c in CASES if gn_path(*c[1:6]) != 'fallback' and gn_path(*c[1:6])[2] == 2}
    assert vec2_cpg >= {10, 30}, vec2_cpg
    # the VAE at 512 x 512 takes the fallback for its full-resolution layers
    assert gn_path(1, 262144, 128, 160, 128) == 'fallback' and gn_path(2, 262144, 256, 320, 256) == 'fallback'
    print(f'{num_sms()} SMs:', sorted(map(str, paths)))


@pytest.mark.parametrize('case', CASES, ids=[_label(c) for c in CASES])
def test_groupnorm_forward(cuda, gn_mode, case):
    """rel-L2 against float64, NaN pad columns of x unread, nothing written outside y's [B*HW, C] window, and two identical
    calls bit-identical."""
    name, B, HW, C, ldx, ldy, dtype, silu, eps = case
    x = _input(B, HW, C, ldx, dtype, cuda, seed=len(name) + B + C)
    gamma, beta = _affine(C, cuda)
    buf, y, ws = _run(x, gamma, beta, B, HW, C, ldy, dtype, eps, silu)
    path = _expected(gn_mode, B, HW, C, ldx, ldy)
    assert untouched(ws, torch.zeros_like(ws, dtype=torch.bool)) == (path != 'fallback'), path   # the path taken
    e = rel_l2(y, _reference(x, C, gamma, beta, eps, silu))
    print(f'GN {_label(case)} [{gn_mode}: {path}] rel-L2 {e:.2e}')
    assert torch.isfinite(y).all()
    assert e < TOL[dtype]
    assert untouched(buf, _window(buf, B, HW, C))
    buf2, _, _ = _run(x, gamma, beta, B, HW, C, ldy, dtype, eps, silu)
    assert same_bits(buf, buf2)


@pytest.mark.parametrize('case', CASES, ids=[_label(c) for c in CASES])
def test_paths_agree(cuda, case):
    """The cluster kernel and the fallback on the same input agree within the output dtype's bound."""
    name, B, HW, C, ldx, ldy, dtype, silu, eps = case
    x = _input(B, HW, C, ldx, dtype, cuda, seed=7)
    gamma, beta = _affine(C, cuda, seed=8)
    _, y_auto, _ = _run(x, gamma, beta, B, HW, C, ldy, dtype, eps, silu)
    with forced_fallback():
        _, y_fb, _ = _run(x, gamma, beta, B, HW, C, ldy, dtype, eps, silu)
    assert rel_l2(y_auto, y_fb) < TOL[dtype]


OFFSET_SHAPES = [('vae', 1, 262144, 128, 160, 128, 1e-6), ('vae', 2, 65536, 256, 320, 256, 1e-6),
                 ('unet', 2, 4096, 320, 320, 320, 1e-5), ('unet', 2, 64, 1280, 1280, 1280, 1e-5)]


@pytest.mark.parametrize('ratio', [0, 10, 30, 100])
@pytest.mark.parametrize('dtype', [BF, H16], ids=['bf16', 'fp16'])
@pytest.mark.parametrize('shape', OFFSET_SHAPES, ids=[_label(s[:6]) for s in OFFSET_SHAPES])
def test_groupnorm_offset(cuda, gn_mode, shape, dtype, ratio):
    """Groups whose mean is `ratio` x their std: the statistics must not lose the variance to cancellation."""
    name, B, HW, C, ldx, ldy, eps = shape
    x = _input(B, HW, C, ldx, dtype, cuda, ratio=float(ratio), seed=3)
    gamma, beta = _affine(C, cuda, seed=4)
    _, y, _ = _run(x, gamma, beta, B, HW, C, ldy, dtype, eps, True)
    e = rel_l2(y, _reference(x, C, gamma, beta, eps, True))
    print(f'GN offset {ratio:>3} {"bf16" if dtype == BF else "fp16"} {_label(shape[:6])} '
          f'[{gn_mode}: {_expected(gn_mode, B, HW, C, ldx, ldy)}] rel-L2 {e:.2e}')
    assert e < TOL[dtype]


OUTLIER_SHAPES = [('unet', 2, 4096, 320, 320, 320, 1e-5), ('vae', 1, 262144, 128, 160, 128, 1e-6),
                  ('vae', 2, 65536, 256, 320, 256, 1e-6)]


@pytest.mark.parametrize('K', [30, 100, 300, 'max'])
@pytest.mark.parametrize('layout', ['pivot', 'corner'])
@pytest.mark.parametrize('dtype', [BF, H16], ids=['bf16', 'fp16'])
@pytest.mark.parametrize('shape', OUTLIER_SHAPES, ids=[_label(s[:6]) for s in OUTLIER_SHAPES])
def test_groupnorm_outlier_pivot(cuda, gn_mode, shape, dtype, layout, K):
    """The element the statistics used to be pivoted on (the group's first element in the sample's first row), or the
    whole first pixel, lies far from its group's mean: the variance must not be lost to cancellation against it.  Held to
    the offset bounds in every (sample, group), not only over the whole tensor."""
    name, B, HW, C, ldx, ldy, eps = shape
    x, _ = plant_outlier(_input(B, HW, C, ldx, dtype, cuda, seed=11), C, layout, K, seed=12)
    gamma, beta = _affine(C, cuda, seed=13)
    _, y, _ = _run(x, gamma, beta, B, HW, C, ldy, dtype, eps, True)
    e = worst_group_rel_l2(y, _reference(x, C, gamma, beta, eps, True), C)
    print(f'GN outlier {layout:6} K={K!s:>3} {"bf16" if dtype == BF else "fp16"} {_label(shape[:6])} '
          f'[{gn_mode}: {_expected(gn_mode, B, HW, C, ldx, ldy)}] worst group rel-L2 {e:.2e}')
    assert torch.isfinite(y).all()
    assert e < TOL[dtype]


@pytest.mark.parametrize('dtype', [BF, H16], ids=['bf16', 'fp16'])
@pytest.mark.parametrize('shape', [(2, 4096, 320, 320, 320), (1, 262144, 128, 160, 128), (3, 288, 960, 960, 960)],
                         ids=['unet', 'vae', 'k4'])
def test_groupnorm_constant_groups(cuda, gn_mode, shape, dtype):
    """Every group is one value (std 0, means up to ~110): the output is act(beta) up to the output rounding, no NaN."""
    B, HW, C, ldx, ldy = shape
    x = _input(B, HW, C, ldx, dtype, cuda, ratio=100.0, seed=5, const=True)
    gamma, beta = _affine(C, cuda, seed=6)
    for silu in (False, True):
        _, y, _ = _run(x, gamma, beta, B, HW, C, ldy, dtype, 1e-6, silu)
        want = (F.silu(beta) if silu else beta).to(dtype).float().expand(B, HW, C)
        assert torch.isfinite(y).all()
        ulp = 2.0 ** (-8 if dtype == BF else -11)
        assert ((y.float() - want).abs() <= 2 * ulp * want.abs() + 1e-3).all(), (y.float() - want).abs().max().item()


@pytest.mark.parametrize('B,HW,C,ldx', [(1, 4096, 320, 320), (2, 65536, 128, 160), (2, 1000, 640, 1280)])
def test_fallback_workspace_capacity(cuda, B, HW, C, ldx):
    """The fallback splits each sample's rows into as many chunks as the fp32 workspace holds (B x 64 floats each):
    exactly B*64 floats gives one chunk, more gives more; B*592*64 is what the engines pass.  Nothing is written past the
    capacity, and B*64 - 1 floats is rejected on the host."""
    from mos_b200 import ops
    dtype = H16
    x = _input(B, HW, C, ldx, dtype, cuda, ratio=3.0, seed=9)
    gamma, beta = _affine(C, cuda, seed=10)
    ref = _reference(x, C, gamma, beta, 1e-6, True)
    outs = []
    with forced_fallback():
        for cap in (B * 64, B * 64 * 3, B * 592 * 64):
            ws = canary((cap + 256,), cuda, torch.float32)
            _, y, _ = _run(x, gamma, beta, B, HW, C, C, dtype, 1e-6, True, partial=ws[:cap])
            assert untouched(ws, window_mask(ws, slice(0, cap)))
            assert rel_l2(y, ref) < TOL[dtype], cap
            outs.append(y.clone())
        y = torch.empty(B, HW, C, device=cuda, dtype=dtype)
        with pytest.raises(ValueError):
            ops.groupnorm(x, gamma, beta, y, torch.zeros(B * 64 - 1, device=cuda), B=B, HW=HW, C=C, eps=1e-6, silu=True,
                          ldx=ldx, ldy=C)
    # one chunk and several chunks sum in different orders: the outputs agree to the bound, not bitwise
    assert rel_l2(outs[0], outs[2]) < TOL[dtype]
