"""Every gradient-fusion solver launch of real fusion walks, audited one by one (tests/solver_audit.py): a float64 reference
with a derived per-element bound, the write window, unchanged operands and a bit-identical second launch; for the
native L-BFGS driver the solve-level checks (bit-identical to the Python driver, the returned loss, no increase).

The walks (tests/engine_walks.py) run on both drivers: the native one (csrc/lbfgs.cu, one mos_lbfgs_solve_batch per
stage) and the Python one (gradient_fusion.FUSION_NATIVE = False, one worker), whose vector launches are audited one by
one.  They are update_quasi_newton and merge_lora_into_weight on the golden cases, the cross-attention K / V stage at the
SD1.5 widths, the text-encoder stage with a CLIPEncoderLayer LoRA, the tiny whole-block spatial stage, and the two
largest SD1.5 solves at 3 iterations.  The last test prints one row per path key and requires the keys reached to be
exactly PATH_KEYS.  The 32 x 64 and 64 x 128 tiles of dgemm_mixed are selected once per process (MOS_DGEMM_TILE), so
they run in a child process each.
"""
import os
import subprocess
import sys
import time

import pytest
import torch

import engine_walks as walks
import solver_audit as sa

pytestmark = pytest.mark.gpu

# The path keys (solver_audit.solver_path) the walks reach, by call site:
#   gradient_fusion.py update_quasi_newton: gram_small / atb_small over the golden K [30, 64] and [400, 48] (row tails
#     of the 16-row tile), vec_dot of V;
#   merge_lora_into_weight / _merged: lora_merge;
#   merge_kv_in_cross_attention / merge_text_encoder: gram_small, sgemm_nn (beta = 0), vec_axpby (beta = 1);
#   GramRecorder (merge_spatial_attention): transpose_bf16 (the tiny UNet's activations: whole 32-row tiles, dense rows;
#     row / column tails and strided rows are audited by test_tail_shapes_audited);
#   solve_from_gram / solve_all: lbfgs_solve_batch with min(8, jobs) workers: 1 for a single solve (golden), 2 for the
#     SD1.5 pair, 4 for the four cross-attention K / V layers, 8 for the text-encoder and spatial stages;
#   lbfgs_minimize (the Python driver): dgemm_mixed, ls_grad_loss, the vector primitives, lbfgs_direction (the walks stop
#     before the history holds 25 pairs; a full, wrapped history is audited in test_solver_audit.py and held bit-identical
#     to the host-driven recursion in test_fusion_gpu.py).
# Outputs rounded once (ls_grad_loss's grad, lora_merge, vec_axpby, vec_absmax) reach err/bound close to 1 by
# construction: their bound is the half-ulp u |result| of that rounding.
PATH_KEYS = {
    'atb_small',
    'atb_small|ntail',
    'dgemm_mixed|64x64',
    'gram_small',
    'gram_small|ntail',
    'lbfgs_direction|k<25',
    'lbfgs_solve_batch|workers=1',
    'lbfgs_solve_batch|workers=2',
    'lbfgs_solve_batch|workers=4',
    'lbfgs_solve_batch|workers=8',
    'lora_merge',
    'ls_grad_loss',
    'sgemm_nn|beta0',
    'transpose_bf16',
    'vec_absmax',
    'vec_absmax|scaled',
    'vec_asum',
    'vec_axpby|beta0',
    'vec_axpby|beta1',
    'vec_dot',
}

STATS = sa.Stats()
T0 = time.time()


def _audit(determinism='all'):
    return lambda: sa.Recorder(STATS, determinism=determinism)


@pytest.fixture(params=['native', 'python'])
def driver(request, monkeypatch):
    import gradient_fusion as gf
    if request.param == 'python':
        monkeypatch.setattr(gf, 'FUSION_NATIVE', False)
        monkeypatch.setattr(gf, 'FUSION_WORKERS', 1)       # the audit follows one host thread
    return request.param


def test_golden(cuda, driver):
    walks.fusion_golden(_audit())


def test_cross_kv_sd15_widths(cuda, driver):
    walks.fusion_cross_kv(_audit('first'))


def test_text_encoder_clip_encoder_layer(cuda, driver):
    walks.fusion_text_encoder(_audit('first'))


def test_spatial_whole_block_tiny(cuda, driver):
    walks.fusion_spatial_whole_block_tiny(_audit('first'))


def test_sd15_solves(cuda, driver):
    out = walks.fusion_sd15_solves(_audit('first'))
    assert set(out) == {'ff.net.0.proj', 'ff.net.2'}


_TILE_CHILD = r'''
import re
import sys
sys.path[:0] = [sys.argv[1], sys.argv[2]]
import torch
from torch.profiler import ProfilerActivity, profile
import solver_audit as sa
from mos_b200 import ops
st = sa.Stats()
with profile(activities=[ProfilerActivity.CUDA]) as prof:
    for M, K, N in ((100, 70, 130), (320, 768, 768), (1280, 1280, 1280), (10240, 1280, 1280)):
        g = torch.Generator(device='cuda').manual_seed(M + K)
        A = torch.randn(M, K, device='cuda', generator=g)
        B = torch.randn(K, N, device='cuda', dtype=torch.float64, generator=g)
        with sa.Recorder(st):
            ops.dgemm_mixed(A, B, torch.empty(M, N, device='cuda', dtype=torch.float64))
            torch.cuda.synchronize()
print(st.table())
assert not st.failures, st.failures
assert set(st.rows) == {'dgemm_mixed|' + sys.argv[3]}, set(st.rows)
# the instantiation the library launched, from the kernel names the profiler saw (demangled or mangled)
tm, tn = sys.argv[3].split('x')
want = re.compile(r'dgemm_mixed_kernel<%s, ?%s>|dgemm_mixed_kernelILi%sELi%sE' % (tm, tn, tm, tn))
names = {e.key for e in prof.key_averages() if 'dgemm_mixed_kernel' in e.key}
print(sorted(names))
assert names and all(want.search(n) for n in names), names
'''


@pytest.mark.parametrize('env,tile', [('1', '32x64'), ('3', '64x128')])
def test_dgemm_mixed_other_tiles(cuda, env, tile):
    """the tiles MOS_DGEMM_TILE selects (read once per process): a child process each, audited at the closure shapes.
    The outputs do not depend on the tile by design, so the child also checks, from the kernel names torch.profiler
    records, that every dgemm launch ran the selected instantiation"""
    here = os.path.dirname(os.path.abspath(__file__))
    pkg = os.path.join(os.path.dirname(here), 'mix-of-show_b200')
    r = subprocess.run([sys.executable, '-c', _TILE_CHILD, here, pkg, tile], capture_output=True, text=True,
                       env=dict(os.environ, MOS_DGEMM_TILE=env), timeout=600)
    print(r.stdout[-3000:])
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]


@pytest.mark.parametrize('bad', ['nan_in_G', 'inf_in_R'])
def test_non_finite_solve_raises_on_both_drivers(cuda, bad):
    """a solve that never sees a finite loss fails (no fused weight from uninitialised memory), names the problem, and
    leaves the caller's buffers untouched"""
    import gradient_fusion as gf
    from mos_b200 import ops
    g = torch.Generator().manual_seed(3)
    K = torch.randn(40, 24, generator=g).cuda()
    W0 = torch.randn(16, 24, generator=g).cuda()
    G, Cm = (K.t() @ K).contiguous(), (W0 @ (K.t() @ K)).contiguous()
    if bad == 'nan_in_G':
        G[3, 5] = float('nan')
    else:
        Cm[7, 2] = float('inf')
    G0, Cm0, W00 = G.clone(), Cm.clone(), W0.clone()
    for native in (True, False):
        with pytest.raises(ValueError, match='finite'):
            gf.solve_from_gram(G, Cm, 1.0, 40, W0, 10, native=native)
    _, Gd, Rd, s, f0 = gf._gram_setup(G, Cm, 1.0, 40, W0)
    ok = gf._gram_setup(G0.nan_to_num(0.0), Cm0.nan_to_num(0.0, 0.0, 0.0), 1.0, 40, W0)
    best = [torch.full((16 * 24,), 7.0, device='cuda') for _ in range(2)]
    with pytest.raises(ValueError, match='problem 1'):
        ops.lbfgs_solve_batch([(ok[1], ok[2], ok[3], ok[4], best[0]), (Gd, Rd, s, f0, best[1])], 10, workers=1)
    assert (best[1] == 7.0).all()
    for t, t0 in ((G, G0), (Cm, Cm0), (W0, W00)):
        assert torch.equal(t.view(torch.int32), t0.view(torch.int32))


def test_tail_shapes_audited(cuda):
    """audited direct calls at the tails the walks above do not reach, on the kernels themselves: the Gram recorder's
    transpose at the lowest UNet level of a 64 x 48 latent (48 rows, a row tail of the 32-row tile) read from a column
    slice (ldx > C) with a column tail, into a padded output; gram_small / atb_small at CLIP fc1 / fc2 widths over row
    counts that end in a partial 16-row tile; the reductions at the ff.net.0.proj size (13.1 M elements)"""
    from mos_b200 import ops
    st = sa.Stats()
    g = torch.Generator(device='cuda').manual_seed(5)
    buf = torch.randn(77, 2 * 1280 + 64, device='cuda', generator=g).to(torch.bfloat16)
    n = 10240 * 1280
    a, b = torch.randn(n, device='cuda', generator=g), torch.randn(n, device='cuda', generator=g)
    out, scratch = torch.zeros(4, device='cuda'), torch.empty(256, device='cuda')
    with sa.Recorder(st):
        for rows, C in ((48, 1280), (77, 1245)):
            x = buf[:rows, 64:64 + C]
            ops.transpose_bf16(x, torch.full((C, rows + 5), 3.0, device='cuda', dtype=torch.bfloat16), rows=rows, C=C,
                               ldx=x.stride(0))
        X = torch.randn(333, 3072, device='cuda', generator=g)
        ops.gram_small(X, torch.randn(3072, 3072, device='cuda', generator=g), accumulate=True)
        ops.atb_small(torch.randn(333, 768, device='cuda', generator=g), X, torch.empty(768, 3072, device='cuda'))
        ops.vec_dot(a, b, out[0:1], scratch)
        ops.vec_asum(a, out[1:2], scratch)
        ops.vec_absmax(a, out[2:3], scratch, 0.5)
        torch.cuda.synchronize()
    print('\n' + st.table())
    assert not st.failures, '\n'.join(st.failures[:30])
    assert set(st.rows) == {'transpose_bf16|rtail|strided', 'transpose_bf16|rtail|ctail|strided', 'gram_small|ntail|acc',
                            'atb_small|ntail', 'vec_dot', 'vec_asum', 'vec_absmax|scaled'}, set(st.rows)


def test_absmax_propagates_nan(cuda):
    """vec_absmax keeps a NaN wherever it sits: in a thread's strided loop, in any warp, block or partial"""
    from mos_b200 import ops
    n = 10240 * 1280
    out, scratch = torch.zeros(1, device='cuda'), torch.empty(256, device='cuda')
    for pos in (0, 31, 255 * 256 + 17, 65536 * 3 + 70000, n - 1):
        a = torch.randn(n, device='cuda')
        a[pos] = float('nan')
        ops.vec_absmax(a, out, scratch, 0.5)
        assert torch.isnan(out).all(), pos
    ops.vec_absmax(a.nan_to_num(0.0), out, scratch, 0.5)
    assert out.item() == (a.nan_to_num(0.0) * 0.5).abs().max().item()


def test_coverage_table(cuda):
    p = torch.cuda.get_device_properties(0)
    print(f'\nsolver launch audit ({time.time() - T0:.0f} s, {p.name}, {p.multi_processor_count} SMs)\n' + STATS.table())
    assert not STATS.failures, '\n'.join(STATS.failures[:30])
    reached = set(STATS.rows)
    assert reached == PATH_KEYS, (f'reached but not listed: {sorted(reached - PATH_KEYS)}; '
                                  f'listed but not reached: {sorted(PATH_KEYS - reached)}')
