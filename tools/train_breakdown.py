"""Differential timing of one captured ED-LoRA training step (forward + loss + backward, TrainEngine): the CUDA graph is
re-captured with one op family replaced by a no-op at a time.  (PDL lets neighbours overlap slightly, so the parts do not
sum exactly to the whole.)   python tools/train_breakdown.py [--batch 4]"""
import argparse
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, 'mix-of-show_b200')]
import torch  # noqa: E402

from mos_b200 import ops  # noqa: E402
from mos_b200.engine import ehs_to_layer_major  # noqa: E402
from mos_b200.train_engine import TrainEngine  # noqa: E402
import bench  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument('--batch', type=int, default=4)
a = ap.parse_args()
B = a.batch
sd, lora = bench.build_workload(False)[:2]
eng = TrainEngine(sd, B, 64, 64, lora=lora, attn_reg_weight=0.01)
g = torch.Generator().manual_seed(100)
x0 = torch.randn(B, 4, 64, 64, generator=g).cuda()
noise = torch.randn(B, 4, 64, 64, generator=g).cuda()
t = torch.randint(0, 1000, (B,), generator=g).cuda()
ehs = ehs_to_layer_major(torch.randn(B, 16, 77, 768, generator=g).cuda())
masks = torch.zeros(B, 1, 64, 64)
masks[:, :, 12:50, 16:44] = 1.0
masks = masks.cuda()
pos = [[4, 5]] * B

FAMILIES = {
    'gemm (fwd+bwd wgmma GEMM/conv)': ['gemm'],
    'splitk_finalize': ['splitk_finalize'],
    'attention fwd': ['attention_train'],
    'attention bwd (+delta)': ['attention_bwd', 'attn_delta'],
    'heads_transpose': ['heads_transpose'],
    'groupnorm fwd': ['groupnorm'],
    'groupnorm bwd': ['groupnorm_bwd'],
    'layernorm fwd': ['layernorm'],
    'layernorm bwd': ['layernorm_bwd'],
    'geglu fwd+bwd': ['geglu_fwd', 'geglu_bwd'],
    'lora_grad': ['lora_grad'],
    'add_rows / resample / im2col': ['add_rows', 'im2col_s2', 'col2im_s2', 'upsample2x', 'upsample2x_bwd'],
    'loss + regulariser': ['masked_mse', 'attn_reg_group', 'attn_reg_total', 'attn_reg_grad'],
}
orig = {n: getattr(ops, n) for names in FAMILIES.values() for n in names}


def noop(*args, **kw):
    return args[3] if len(args) > 3 else None


def timeit(skip_names, reps=5):
    for n, f in orig.items():
        setattr(ops, n, noop if n in skip_names else f)
    eng._tgraphs = {}
    eng.tgraph = None
    for _ in range(2):
        eng.forward_backward(x0, noise, t, ehs, masks, token_pos=pos)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        eng.forward_backward(x0, noise, t, ehs, masks, token_pos=pos)
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


full = timeit([])
print(f'full forward+loss+backward graph, batch {B}: {full:8.3f} ms')
for fam, names in FAMILIES.items():
    tt = timeit(names)
    print(f'  without {fam:36s} {tt:8.3f} ms  -> ~ {full - tt:7.3f} ms ({100 * (full - tt) / full:4.1f} %)')
