"""Numerics experiment on the fp32 CPU oracle (test infrastructure; not collected by pytest, not a product path).

Emulates WHERE the GPU engine rounds (GEMM operands, weights, stored intermediates, the residual stream) by running
the oracle UNet with rounding functions inserted at the same points, and prints the eps error and the post-scheduler
latent error (guidance 1 and 7.5) against the un-rounded fp32 oracle.  It answered the round-2 design question "what has
to stay fp32 for the CFG-7.5 latents to meet 1e-3" (answer: fp16 operands; see DESIGN.md "Numerics").

    python tests/numerics_emulation.py [--full] [--modes a,b,...]
"""
import argparse
import os
import sys
import types

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import edlora_ref as er  # noqa: E402
from oracle import inject  # noqa: E402
from oracle import unet as ou  # noqa: E402
from oracle.schedulers import DPMSolverMultistepScheduler  # noqa: E402


def bf16(x):
    return x.to(torch.bfloat16).float()


def fp16(x):
    return x.to(torch.float16).float()


def ident(x):
    return x


class Cfg:
    def __init__(self, rw=ident, ra=ident, ri=ident, rs=ident):
        self.rw, self.ra, self.ri, self.rs = rw, ra, ri, rs


C = Cfg()


def lin(m, x):
    """GEMM with rounded operands, fp32 accumulation, fp32 bias; LoRA (inject.py patches m.forward) kept as installed."""
    if isinstance(m, torch.nn.Conv2d):
        y = F.conv2d(C.ra(x), C.rw(m.weight), m.bias, m.stride, m.padding)
    else:
        y = F.linear(C.ra(x), C.rw(m.weight), m.bias)
    lora = getattr(m, '_emul_lora', None)
    if lora is not None:
        d, u, alpha = lora
        y = y + alpha * F.linear(F.linear(C.ra(x), bf16(d)), u)
    return y


def resnet_fwd(self, x, temb):
    n1 = F.silu(self.norm1(x))
    h = lin(self.conv1, n1) + self.time_emb_proj(F.silu(temb))[:, :, None, None]
    h = C.ri(h)
    n2 = F.silu(self.norm2(h))
    sc = x
    if self.conv_shortcut is not None:
        sc = C.ri(lin(self.conv_shortcut, x))
    return C.rs(lin(self.conv2, n2) + sc)


def attn_core(attn, x, ctx):
    q = C.ri(lin(attn.to_q, x))
    k = C.ri(lin(attn.to_k, ctx))
    v = C.ri(lin(attn.to_v, ctx))
    q, k, v = (attn.head_to_batch_dim(t) for t in (q, k, v))
    if q.shape[1] > 1024 and k.shape[1] > 1024:
        o = F.scaled_dot_product_attention(q, k, v, scale=attn.scale)
    else:
        p = (torch.bmm(q, k.transpose(1, 2)) * attn.scale).softmax(-1)
        o = torch.bmm(C.ra(p), v)
    o = C.ri(attn.batch_to_head_dim(o))
    return lin(attn.to_out[0], o)


def block_fwd(self, x, encoder_hidden_states=None, cross_attention_kwargs=None):
    x = C.rs(attn_core(self.attn1, self.norm1(x), self.norm1(x)) + x)
    ehs = encoder_hidden_states
    idx = self.attn2.processor.cross_attention_idx if hasattr(self.attn2.processor, 'cross_attention_idx') else None
    if ehs.ndim == 4:
        ehs = ehs[:, idx]
    x = C.rs(attn_core(self.attn2, self.norm2(x), ehs) + x)
    proj = self.ff.net[0].proj
    a, g = lin(proj, self.norm3(x)).chunk(2, dim=-1)
    ff = C.ri(a * F.gelu(g))
    return C.rs(lin(self.ff.net[2], ff) + x)


def tr_fwd(self, x, encoder_hidden_states=None, cross_attention_kwargs=None):
    b, c, h, w = x.shape
    res = x
    x = C.rs(lin(self.proj_in, self.norm(x)))
    x = x.permute(0, 2, 3, 1).reshape(b, h * w, -1)
    for blk in self.transformer_blocks:
        x = blk(x, encoder_hidden_states, cross_attention_kwargs)
    x = x.reshape(b, h, w, -1).permute(0, 3, 1, 2).contiguous()
    return C.rs(lin(self.proj_out, x) + res)


def down_fwd(self, x):
    return C.rs(lin(self.conv, x))


def up_fwd(self, x, output_size=None):
    if output_size is not None:
        return C.rs(lin(self.conv, F.interpolate(x, size=output_size, mode='nearest')))
    return C.rs(lin(self.conv, F.interpolate(x, scale_factor=2.0, mode='nearest')))


def patch(unet, lora):
    for name, m in unet.named_modules():
        cn = m.__class__.__name__
        if cn == 'ResnetBlock2D':
            m.forward = types.MethodType(resnet_fwd, m)
        elif cn == 'BasicTransformerBlock':
            m.forward = types.MethodType(block_fwd, m)
        elif cn == 'Transformer2DModel':
            m.forward = types.MethodType(tr_fwd, m)
        elif cn == 'Downsample2D':
            m.forward = types.MethodType(down_fwd, m)
        elif cn == 'Upsample2D':
            m.forward = types.MethodType(up_fwd, m)
        if lora is not None and name + '.lora_down.weight' in lora:
            d = lora[name + '.lora_down.weight']
            u = lora[name + '.lora_up.weight']
            m._emul_lora = (d.reshape(d.shape[0], -1), u.reshape(u.shape[0], -1), 1.0)
    orig_in, orig_out = unet.conv_in.forward, unet.conv_out.forward
    unet.conv_in.forward = lambda x: C.rs(orig_in(x))


MODES = {
    'fp32': Cfg(),
    'r1 (bf16 everything)': Cfg(bf16, bf16, bf16, bf16),
    'bf16 ops+w+interm, fp32 residual': Cfg(bf16, bf16, bf16, ident),
    'bf16 ops+w, fp32 interm+residual': Cfg(bf16, bf16, ident, ident),
    'fp16 ops+interm, bf16 w, fp32 residual': Cfg(bf16, fp16, fp16, ident),
    'fp16 ops+interm+w, fp32 residual': Cfg(fp16, fp16, fp16, ident),
    'fp16 everything': Cfg(fp16, fp16, fp16, fp16),
    'fp16 acts+interm+residual, bf16 w': Cfg(bf16, fp16, fp16, fp16),
    'residual only bf16': Cfg(ident, ident, ident, bf16),
    'weights only bf16': Cfg(bf16, ident, ident, ident),
    'operands only bf16': Cfg(ident, bf16, ident, ident),
    'interm only bf16': Cfg(ident, ident, bf16, ident),
}


def main():
    global C
    ap = argparse.ArgumentParser()
    ap.add_argument('--full', action='store_true')
    ap.add_argument('--hw', type=int, default=0)
    ap.add_argument('--modes', default='')
    args = ap.parse_args()
    cfg = None if args.full else ou.TINY
    H = W = args.hw or (64 if args.full else 32)
    unet = ou.build_unet(0, cfg)
    inject.install_edlora_processors(unet)
    lora = inject.random_lora_state(unet, seed=10)
    patch(unet, lora)
    lat1 = torch.randn(1, 4, H, W, generator=torch.Generator().manual_seed(1))
    ehs = torch.randn(2, 16, 77, 768, generator=torch.Generator().manual_seed(2))
    sched = DPMSolverMultistepScheduler()
    sched.set_timesteps(50)
    t0 = int(sched.timesteps[0])
    lat2 = torch.cat([lat1, lat1])
    ref = None
    sel = [m for m in MODES if not args.modes or any(s in m for s in args.modes.split(','))]
    if 'fp32' not in sel:
        sel = ['fp32'] + sel
    for name in sel:
        C = MODES[name]
        with torch.no_grad():
            eps = unet(lat2, torch.tensor([t0, t0]), ehs).sample
        s1 = DPMSolverMultistepScheduler()
        s1.set_timesteps(50)
        l75 = s1.step(er.cfg_combine(eps, 7.5), t0, lat1).prev_sample
        s2 = DPMSolverMultistepScheduler()
        s2.set_timesteps(50)
        l1 = s2.step(eps[1:], t0, lat1).prev_sample
        if ref is None:
            ref = (eps, l1, l75)
            continue
        r = lambda a, b: ((a - b).norm() / b.norm()).item()
        print(f'{name:45s} eps {r(eps, ref[0]):.2e}  latents g=1 {r(l1, ref[1]):.2e}  g=7.5 {r(l75, ref[2]):.2e}',
              flush=True)


if __name__ == '__main__':
    main()
