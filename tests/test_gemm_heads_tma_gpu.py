"""Head-split output of the wgmma GEMM written by TMA stores (csrc/gemm.cu, `epi_heads`).

Q/K segments ([batch * heads, rows_pad, dpad]) and V^T segments ([batch * heads, dv_pad, rows_pad]) are written from the
staging tile by one tensor map per segment whose extents are head_dim and tokens_per_batch.  Every case here:
- matches the fp32 PyTorch reference (TF32 off; tolerances of test_gemm_schedule_gpu.py);
- leaves the pad columns (head_dim..dpad), the V^T pad rows (head_dim..dv_pad) and the pad tokens (T..rows_pad) holding
  the sentinel they were filled with: the attention kernels multiply the Q/K pad columns;
- is bit-identical to the consumer copy-out path, which MOS_GEMM_HEADS_COPY=1 selects for every launch.  That switch is
  read once per process, so the copy-out outputs come from a child process (this file run as a script) as hashes.

Token counts: 4096, 1024 and 256 (a tile inside one batch), 64 with an odd batch count (a tile spans two batches, the
last tile half outside the output) and 77 (the copy-out fallback: tiles cross batches mid-chunk).
"""
import hashlib
import json
import os
import subprocess
import sys

import pytest
import torch

if __name__ == '__main__':
    _root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    sys.path[:0] = [_root, os.path.join(_root, 'mix-of-show_b200')]

from gpu_helpers import bits, canary, mk, rel_l2, rup, untouched, window_mask  # noqa: E402

pytestmark = pytest.mark.gpu
TOL = {torch.bfloat16: 4e-3, torch.float16: 6e-4}
H = 8                                              # heads
K = 320
SHAPES = [(40, 4096, 1), (80, 1024, 2), (160, 256, 4), (160, 64, 5), (40, 64, 3), (40, 77, 4), (80, 77, 2)]  # (d, T, B)
CASES = [(d, T, B, nseg, dt, lora) for d, T, B in SHAPES for nseg in (1, 3) for dt in ('bf16', 'fp16')
         for lora in (False, True)]
DTYPES = {'bf16': torch.bfloat16, 'fp16': torch.float16}


def _case_id(c):
    d, T, B, nseg, dt, lora = c
    return f'd{d}-T{T}-B{B}-seg{nseg}-{dt}' + ('-lora' if lora else '')


def _run(case, dev):
    """One launch; returns (segment buffers, their kinds, rows_pad list, fp32 reference [B, T, nseg, H, d])."""
    from mos_b200 import ops
    from mos_b200._lib import MOS_SEG_ROWS, MOS_SEG_TRANSPOSED
    d, T, B, nseg, dt, lora = case
    dtype = DTYPES[dt]
    C, dp, dvp = H * d, rup(d, 64), rup(d, 16)
    N, M = nseg * C, B * T
    A = mk((M, K), dev, seed=1, dtype=dtype)
    W = mk((N, K), dev, K ** -0.5, seed=2, dtype=dtype)
    ref = A.float() @ W.float().t()
    kw = {}
    if lora:
        downs = [mk((4, K), dev, K ** -0.5, 10 + s, dtype) for s in range(nseg)]
        up = (torch.randn(N, 4, generator=torch.Generator().manual_seed(110)) * 0.5).to(dev)
        down16 = torch.zeros(16, K, device=dev, dtype=dtype)
        for s in range(nseg):
            down16[4 * s:4 * s + 4] = downs[s]
            ref[:, s * C:(s + 1) * C] += (A.float() @ downs[s].float().t()) @ up[s * C:(s + 1) * C].t()
        kw = dict(lora_down=down16, lora_up=up, lora_seg=C)
    kinds = [MOS_SEG_ROWS] * min(nseg, 2) + [MOS_SEG_TRANSPOSED] * (nseg - 2)
    pads = [T + 5 if k == MOS_SEG_ROWS else rup(T, 8) + 8 for k in kinds]
    segs = [canary((B * H, r, dp), dev, dtype) if k == MOS_SEG_ROWS else canary((B * H, dvp, r), dev, dtype)
            for k, r in zip(kinds, pads)]
    ops.gemm(A, W, None, heads=dict(seg_ptr=segs, seg_kind=kinds, seg_rows_pad=pads, heads=H, head_dim=d, dpad=dp,
                                    dv_pad=dvp, tokens_per_batch=T), **kw)
    torch.cuda.synchronize()
    return segs, kinds, ref.view(B, T, nseg, H, d)


def _digest(segs):
    return [hashlib.sha256(bits(s).cpu().numpy().tobytes()).hexdigest() for s in segs]


@pytest.fixture(scope='module')
def copy_out_digests(cuda, tmp_path_factory):
    """hashes of every case's segment buffers, computed with the copy-out path in a child process"""
    path = tmp_path_factory.mktemp('heads_copy') / 'digests.json'
    env = dict(os.environ, MOS_GEMM_HEADS_COPY='1')
    r = subprocess.run([sys.executable, os.path.abspath(__file__), str(path)], env=env, capture_output=True, text=True)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-4000:]
    with open(path) as f:
        return json.load(f)


@pytest.mark.parametrize('case', CASES, ids=_case_id)
def test_heads_tma(cuda, copy_out_digests, case):
    from mos_b200._lib import MOS_SEG_ROWS
    d, T, B = case[:3]
    dtype = DTYPES[case[4]]
    segs, kinds, ref = _run(case, cuda)
    for s, (buf, kind) in enumerate(zip(segs, kinds)):
        r = ref[:, :, s]
        if kind == MOS_SEG_ROWS:
            got, want = buf[:, :T, :d], r.permute(0, 2, 1, 3).reshape(B * H, T, d)
            win = window_mask(buf, slice(None), slice(0, T), slice(0, d))
        else:
            got, want = buf[:, :d, :T], r.permute(0, 2, 3, 1).reshape(B * H, d, T)
            win = window_mask(buf, slice(None), slice(0, d), slice(0, T))
        e = rel_l2(got, want)
        assert e < TOL[dtype], f'segment {s}: rel-L2 {e:.2e}'
        assert untouched(buf, win), f'segment {s}: write outside the head-split window'
    assert _digest(segs) == copy_out_digests[_case_id(case)], 'TMA stores and copy-out differ'


if __name__ == '__main__':
    torch.backends.cuda.matmul.allow_tf32 = False
    dev = torch.device('cuda:0')
    out = {_case_id(c): _digest(_run(c, dev)[0]) for c in CASES}
    with open(sys.argv[1], 'w') as f:
        json.dump(out, f)
