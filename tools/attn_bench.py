"""Device time of the flash-attention kernel at the shapes of one SD1.5 denoise step (CFG batch 2, 8 heads).
  python tools/attn_bench.py [--batch 2]
Algorithmic FLOPs = 4 * nq * nk * d per (batch, head) (SURVEY.md 8d); time = CUDA events over 20 back-to-back launches."""
import argparse
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, 'mix-of-show_b200')]
import torch  # noqa: E402

from mos_b200 import ops  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument('--batch', type=int, default=2)
ap.add_argument('--reps', type=int, default=20)
a = ap.parse_args()
B, H = a.batch, 8
print(f'batch {B}')
for d, nq, nk in [(40, 4096, 4096), (80, 1024, 1024), (160, 256, 256), (160, 64, 64), (40, 4096, 77), (80, 1024, 77),
                  (160, 256, 77), (40, 18432, 18432)]:
    if nq > 8192 and B > 2:
        continue
    dp, dv, nk8 = (d + 63) // 64 * 64, (d + 15) // 16 * 16, (nk + 7) // 8 * 8
    g = torch.Generator(device='cuda').manual_seed(0)
    Q = torch.zeros(B * H, nq, dp, device='cuda', dtype=torch.bfloat16)
    K = torch.zeros(B * H, nk, dp, device='cuda', dtype=torch.bfloat16)
    Vt = torch.zeros(B * H, dv, nk8, device='cuda', dtype=torch.bfloat16)
    Q[..., :d] = torch.randn(B * H, nq, d, device='cuda', generator=g)
    K[..., :d] = torch.randn(B * H, nk, d, device='cuda', generator=g)
    Vt[:, :d, :nk] = torch.randn(B * H, d, nk, device='cuda', generator=g)
    out = torch.empty(B, nq, H * d, device='cuda', dtype=torch.bfloat16)
    for _ in range(3):
        ops.attention(Q, K, Vt, out, batch=B, heads=H, head_dim=d, nq=nq, nk=nk)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(a.reps):
        ops.attention(Q, K, Vt, out, batch=B, heads=H, head_dim=d, nq=nq, nk=nk)
    e1.record()
    torch.cuda.synchronize()
    us = e0.elapsed_time(e1) / a.reps * 1e3
    fl = 4.0 * nq * nk * d * B * H
    tiles = B * H * -(-nq // 128) * -(-nk // 128)
    print(f'd={d:3d} nq={nq:5d} nk={nk:5d}: {us:9.1f} us  {fl / us / 1e6:7.1f} TFLOP/s (algorithmic)  '
          f'{us * 1e-6 * 1.98e9 * 132 / tiles:7.0f} SM-cycles per 128x128 block')
