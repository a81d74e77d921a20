"""Device time of the flash-attention kernel at the shapes of one SD1.5 denoise step (CFG batch 2, 8 heads).
  python tools/attn_bench.py [--batch 2] [--dtype fp16|bf16]
Algorithmic FLOPs = 4 * nq * nk * d per (batch, head) (SURVEY.md 8d); time = CUDA events over 20 back-to-back launches.
SM-cycles per 128x128 block use the SM clock nvidia-smi reports for this card right after each timed window, next to
two floors per block: MUFU = 128 * 128 ex2 at 16 per clock per SM, tensor = the padded QK^T (k = 16-rounded d) and PV (n = 16-rounded d) FLOPs at the dense
16-bit rate of 4096 FLOP per clock per SM (989 TFLOP/s over 132 SMs at 1.83 GHz)."""
import argparse
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, 'mix-of-show_b200')]
import torch  # noqa: E402

from mos_b200 import ops  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument('--batch', type=int, default=2)
ap.add_argument('--reps', type=int, default=20)
ap.add_argument('--dtype', default='fp16', choices=['fp16', 'bf16'], help='operand type (sampling runs fp16)')
a = ap.parse_args()
B, H = a.batch, 8
dt = torch.float16 if a.dtype == 'fp16' else torch.bfloat16
props = torch.cuda.get_device_properties(torch.cuda.current_device())
GPU_ID = f'GPU-{props.uuid}'   # the card this process runs on, whatever CUDA_VISIBLE_DEVICES maps it to


def smi(fields):
    q = subprocess.run(['nvidia-smi', '-i', GPU_ID, f'--query-gpu={fields}', '--format=csv,noheader,nounits'],
                       capture_output=True, text=True, check=True).stdout.strip()
    return [f.strip() for f in q.split(',')]


name, power, max_mhz = smi('name,power.limit,clocks.max.sm')
sms = props.multi_processor_count
print(f'batch {B}, {a.dtype}, {name}, power limit {power} W, max SM clock {max_mhz} MHz, {sms} SMs; cycles use the SM '
      f'clock sampled right after each timed window')
for d, nq, nk in [(40, 4096, 4096), (80, 1024, 1024), (160, 256, 256), (160, 64, 64), (40, 4096, 77), (80, 1024, 77),
                  (160, 256, 77), (40, 18432, 18432)]:
    if nq > 8192 and B > 2:
        continue
    dp, dv, nk8 = (d + 63) // 64 * 64, (d + 15) // 16 * 16, (nk + 7) // 8 * 8
    g = torch.Generator(device='cuda').manual_seed(0)
    Q = torch.zeros(B * H, nq, dp, device='cuda', dtype=dt)
    K = torch.zeros(B * H, nk, dp, device='cuda', dtype=dt)
    Vt = torch.zeros(B * H, dv, nk8, device='cuda', dtype=dt)
    Q[..., :d] = torch.randn(B * H, nq, d, device='cuda', generator=g)
    K[..., :d] = torch.randn(B * H, nk, d, device='cuda', generator=g)
    Vt[:, :d, :nk] = torch.randn(B * H, d, nk, device='cuda', generator=g)
    out = torch.empty(B, nq, H * d, device='cuda', dtype=dt)
    for _ in range(3):
        ops.attention(Q, K, Vt, out, batch=B, heads=H, head_dim=d, nq=nq, nk=nk)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(a.reps):
        ops.attention(Q, K, Vt, out, batch=B, heads=H, head_dim=d, nq=nq, nk=nk)
    e1.record()
    mhz = float(smi('clocks.sm')[0])
    torch.cuda.synchronize()
    clk = mhz * 1e6
    us = e0.elapsed_time(e1) / a.reps * 1e3
    fl = 4.0 * nq * nk * d * B * H
    tiles = B * H * -(-nq // 128) * -(-nk // 128)
    mufu = 128 * 128 / 16
    tensor = 2 * 128 * 128 * (dv + dv) / 4096
    print(f'd={d:3d} nq={nq:5d} nk={nk:5d}: {us:9.1f} us  {fl / us / 1e6:7.1f} TFLOP/s (algorithmic)  '
          f'{us * 1e-6 * clk * sms / tiles:7.0f} SM-cycles per 128x128 block at {mhz:.0f} MHz  (floors: MUFU '
          f'{mufu:.0f}, tensor {tensor:.0f})')
