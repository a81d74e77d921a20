"""Run the denoise step eagerly (no CUDA graph) a few times: the command ncu wraps for launch lists / full captures.
   ncu --metrics gpu__time_duration.sum --clock-control none -s <skip> -c <n> --csv --log-file out.csv \
       python tools/profile_step.py --runs 2
Prints the number of kernel launches per step so that -s / -c can be chosen."""
import argparse
import os
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, 'mix-of-show_b200')):
    sys.path.insert(0, p)
import torch  # noqa: E402

import bench  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument('--runs', type=int, default=2)
ap.add_argument('--tiny', action='store_true')
ap.add_argument('--merged', action='store_true')
ap.add_argument('--height', type=int, default=64)
ap.add_argument('--width', type=int, default=64)
ap.add_argument('--out', default=os.path.join(tempfile.gettempdir(), 'mos_profile_step'),
                help='directory for gemm_shapes.csv (default: under the system temporary directory)')
args = ap.parse_args()
from mos_b200.engine import UNetEngine, ehs_to_layer_major  # noqa: E402

sd, lora, lat, ehs, cfg = bench.build_workload(args.tiny)
kw = dict(block_out=cfg['block_out_channels'], layers=cfg['layers_per_block']) if cfg else {}
eng = UNetEngine(sd, 2, args.height, args.width, lora=lora, merge_lora=args.merged, use_graph=False, **kw)
nx = len(eng.xattn_names)
eng.in_ehs.copy_(ehs_to_layer_major(ehs[:, :nx].cuda(), nx))
eng.in_latents.normal_()
eng.in_t.fill_(981.0)
for _ in range(args.runs):          # warm-up runs (allocate scratch, set attributes)
    eng._run()
torch.cuda.synchronize()
# log the shape of every wgmma GEMM launch of the profiled step, in launch order (-> <--out>/gemm_shapes.csv), so
# that the per-launch times of the ncu list can be attributed to layer shapes
from mos_b200 import ops  # noqa: E402

shapes = []
_orig = ops.gemm


def _logging_gemm(A, W, out=None, **kw):
    conv = kw.get('conv')
    M = conv[0] * conv[1] * conv[2] if conv is not None else (kw.get('M') or A.shape[0])
    shapes.append((M, W.shape[0], W.shape[1], int(conv is not None), int(kw.get('lora_down') is not None),
                   int(bool(kw.get('geglu'))), int(kw.get('heads') is not None), kw.get('splits') or 1))
    return _orig(A, W, out, **kw)


ops.gemm = _logging_gemm
torch.cuda.profiler.start()         # use with: ncu --profile-from-start off
eng._run()
torch.cuda.synchronize()
torch.cuda.profiler.stop()
ops.gemm = _orig
print('launches per step:', eng.launches)
os.makedirs(args.out, exist_ok=True)
with open(os.path.join(args.out, 'gemm_shapes.csv'), 'w') as f:
    f.write('M,N,K,conv,lora,geglu,heads,splits\n')
    for sh in shapes:
        f.write(','.join(str(v) for v in sh) + '\n')
print('GEMM shapes:', os.path.join(args.out, 'gemm_shapes.csv'))
