"""Training at the batch sizes one H100 runs besides the shipped B = 2: `batch_size_per_gpu: 4`, or 2 with
`gradient_accumulation_steps: 2` (the upstream `..._B4_...` configs give 4 images per step on two GPUs).

- samples do not mix: one B = 4 TrainEngine against a B = 1 engine with the same weights fed each sample alone (per-sample
  eps and MSE terms, and the B = 4 gradient against the mean of the four B = 1 gradients);
- accumulation through EDLoRATrainer (text encoder, concept rows and UNet): two B = 2 micro-batches, the second with
  `accumulate`, scaled by 1/2, against one B = 4 step (regulariser off), then the AdamW step from either; with the
  regulariser on, against the sum of the two micro-batches' fp32 autograd gradients (the reference regularises per
  micro-batch); and through `train_edlora.train(..., gradient_accumulation_steps=2)`;
- the launch audits of the full-size step (SD1.5 at 64 x 64, 12-layer CLIP, regulariser, optimiser step) at B = 4 and 1;
- `train_edlora.py -opt` end to end with `batch_size_per_gpu: 4` and with 2 plus `gradient_accumulation_steps: 2`.

Bounds: eps 2e-2 rel-L2 (the bf16 forward target of test_train_gpu), per-sample MSE terms 1e-3 relative, gradients 4e-2
rel-L2 (the autograd bound of test_trainer_full_gpu).  A sample mix-up or a wrong 1 / B gives errors of order 1."""
import json

import pytest
import torch

import engine_walks as walks
from test_trainer_full_gpu import (FINETUNE, _base_dir, _cos, _delta, _trainer, autograd_reference, batch_inputs,
                                   format_errors, group_errors, rel_l2)

pytestmark = pytest.mark.gpu

GROUPS = ('rows', 'text', 'unet')


def _flat_groups(state, flat):
    """the three groups of a flat gradient [concept rows | text LoRA | UNet LoRA] as (name, slice)"""
    lo = (0,) + tuple(state.group_end[:2])
    return [(name, flat[a:b]) for name, a, b in zip(GROUPS, lo, state.group_end)]


def _compare_flat(state, got, want):
    """{group: (rel-L2, cosine, size)} and the whole flat vector's (rel-L2, cosine)"""
    res = {name: (rel_l2(g, w), _cos(g, w), g.numel())
           for (name, g), (_, w) in zip(_flat_groups(state, got), _flat_groups(state, want))}
    return res, (rel_l2(got, want), _cos(got, want))


# ------------------------------------------------------------------------------------------------ a. samples do not mix
def test_batch4_engine_matches_four_single_sample_steps(cuda):
    """B = 4 TrainEngine (SD1.5 channels, one layer per block, 16 x 16, regulariser off) vs one B = 1 engine with the same
    weights run on each sample (a B = 1 step overwrites the gradient, so one engine serves for the four).

    Both forwards are bf16, and the two batch sizes take different GroupNorm partitions and GEMM split-K slices, so their
    bf16 roundings differ; each is held to the fp32 oracle at the bf16 forward target of test_train_gpu (2e-2), and the
    two to each other at the same bound.  The MSE terms and the gradient carry the sample bookkeeping and 1 / B."""
    from mos_b200.engine import ehs_to_layer_major
    from mos_b200.train_engine import TrainEngine
    from oracle import inject
    from oracle import unet as ou
    from oracle.schedulers import DDPMScheduler
    cfg = dict(block_out_channels=(320, 640, 1280, 1280), layers_per_block=1)
    ref = ou.build_unet(0, cfg)
    lora = inject.random_lora_state(ref, seed=10)
    sd = {k: v.detach().clone() for k, v in ref.state_dict().items()}
    B, H = 4, 16
    g = torch.Generator().manual_seed(7)
    x0, noise = torch.randn(B, 4, H, H, generator=g), torch.randn(B, 4, H, H, generator=g)
    t = torch.tensor([0, 999, 511, 130])
    masks = (torch.rand(B, 1, H, H, generator=g) > 0.5).float()
    masks[B - 1] = 1.0

    def engine(b):
        return TrainEngine(sd, b, H, H, lora=lora, attn_reg_weight=None, block_out=cfg['block_out_channels'], layers=1,
                           use_graph=False)

    def step(eng, sl, ehs):
        eng.forward_backward(x0[sl].cuda(), noise[sl].cuda(), t[sl].cuda(), ehs_to_layer_major(ehs[sl].cuda(), nx),
                             masks[sl].cuda())
        torch.cuda.synchronize()
        return eng.out_eps.cpu().clone(), eng.mse_ws.cpu().clone(), eng.state.grads[:eng.state.n].cpu().clone(), \
            eng.loss_out[0].item()

    big = engine(B)
    nx = len(big.xattn_names)
    ehs = torch.randn(B, nx, 77, 768, generator=g).to(torch.bfloat16).float()
    eps4, ws4, g4, loss4 = step(big, slice(0, B), ehs)
    del big
    torch.cuda.empty_cache()
    one = engine(1)
    g_sum, terms, e_eps, e_mse, eps1 = torch.zeros_like(g4), [], [], [], []
    for b in range(B):
        e1, ws1, g1, _ = step(one, slice(b, b + 1), ehs)
        eps1.append(e1[0])
        e_eps.append(rel_l2(eps4[b], e1[0]))
        mse4, mse1 = (ws4[2 * b] / ws4[2 * b + 1]).item(), (ws1[0] / ws1[1]).item()
        terms.append(mse1)
        e_mse.append(abs(mse4 - mse1) / abs(mse1))
        g_sum += g1
    del one
    torch.cuda.empty_cache()
    inject.install_edlora_processors(ref)
    inject.inject_lora(ref, lora, 1.0)
    with torch.no_grad():                                       # fp32 on the CPU: 4 samples at 16 x 16
        eps_ref = ref(DDPMScheduler().add_noise(x0, noise, t), t, ehs).sample
    o4 = [rel_l2(eps4[b], eps_ref[b]) for b in range(B)]
    o1 = [rel_l2(eps1[b], eps_ref[b]) for b in range(B)]
    e_g, c_g = rel_l2(g4, g_sum / B), _cos(g4, g_sum / B)
    print(f'B=4 vs 4 x B=1: eps rel-L2 {["%.2e" % e for e in e_eps]} (vs fp32 oracle: B=4 {["%.2e" % e for e in o4]}, '
          f'B=1 {["%.2e" % e for e in o1]}); MSE terms {["%.5f" % m for m in terms]} rel err '
          f'{["%.1e" % e for e in e_mse]}; loss {loss4:.6f} vs mean {sum(terms) / B:.6f}; flat gradient rel-L2 {e_g:.3e} '
          f'cos {c_g:.5f}')
    assert max(o4) < 2e-2 and max(o1) < 2e-2
    assert max(e_eps) < 2e-2
    assert max(e_mse) < 1e-3
    assert abs(loss4 - sum(terms) / B) < 1e-3 * abs(loss4)
    assert e_g < 4e-2


# ------------------------------------------------------------------------------------------------ b. accumulation
def _fixed(n_micro, seed=60):
    """four samples (batch_inputs(4)) as n_micro micro-batches of 4 / n_micro, with their noise and timesteps"""
    prompts, lat, noise, t, masks = batch_inputs(4, seed=seed)
    k = 4 // n_micro
    return [dict(images=lat[i:i + k], prompts=prompts[i:i + k], masks=masks[i:i + k],
                 img_masks=torch.ones_like(masks[i:i + k]), noise=noise[i:i + k], timesteps=t[i:i + k])
            for i in range(0, 4, k)]


def _step(tr, mb, accumulate=False):
    return tr(mb['images'], mb['prompts'], mb['masks'], mb['img_masks'], noise=mb['noise'], timesteps=mb['timesteps'],
              accumulate=accumulate)


def _adamw_reference(p0, grad, lrs, group_end):
    """torch.optim.AdamW (weight decay 0.01) from p0 on grad, one step, the three learning-rate groups"""
    lo = (0,) + tuple(group_end[:2])
    leaves = [p0[a:b].clone().requires_grad_(True) for a, b in zip(lo, group_end)]
    opt = torch.optim.AdamW([{'params': [p], 'lr': lr} for p, lr in zip(leaves, lrs)], weight_decay=0.01)
    for p, a, b in zip(leaves, lo, group_end):
        p.grad = grad[a:b].clone()
    opt.step()
    return torch.cat([p.detach() for p in leaves])


def test_accumulation_matches_batch4_step(cuda, tmp_path):
    """regulariser off: two B = 2 micro-batches (`accumulate` on the second) x 1/2 == one B = 4 step, all three groups;
    then AdamW from the same state on each (grad_scale 1 and 1/2) follows torch.optim.AdamW on its own gradient"""
    from test_fusion_orchestration import WordTokenizer
    from mos_b200 import dp
    base, ref_unet, clip = _base_dir(tmp_path)
    delta = _delta(ref_unet, clip)
    one, two = _trainer(base, WordTokenizer(), None, False), _trainer(base, WordTokenizer(), None, False)
    for tr in (one, two):
        tr.load_delta_state_dict(delta)
    (b4,) = _fixed(1)
    _step(one, b4)
    for k, mb in enumerate(_fixed(2)):
        _step(two, mb, accumulate=k > 0)
    torch.cuda.synchronize()
    n = one.state.n
    assert two.state.n == n and torch.equal(one.state.params, two.state.params)
    g4, g22 = one.state.grads[:n].cpu().clone(), two.state.grads[:n].cpu().clone()
    res, (e, c) = _compare_flat(one.state, g22 / 2, g4)
    print(f'accumulated 2 x B=2 / 2 vs B=4: flat rel-L2 {e:.3e} cos {c:.5f};  ' + format_errors(res))
    assert e < 4e-2
    for name, (r, cos, _) in res.items():
        assert r < 4e-2 and cos > 0.998, name
    p0 = one.state.params.cpu().clone()
    dp.optimizer_step(one.state, 1.0)
    dp.optimizer_step(two.state, 0.5)
    torch.cuda.synchronize()
    p4, p22 = one.state.params.cpu(), two.state.params.cpu()
    e_opt = [rel_l2(p - p0, _adamw_reference(p0, gr * s, one.state.lrs, one.state.group_end) - p0)
             for p, gr, s in ((p4, g4, 1.0), (p22, g22, 0.5))]
    print(f'after one AdamW step: params rel-L2 {rel_l2(p22, p4):.3e} (update cos {_cos(p22 - p0, p4 - p0):.4f}); '
          f'updates vs torch.optim.AdamW {e_opt[0]:.1e} / {e_opt[1]:.1e}')
    assert max(e_opt) < 1e-5
    assert rel_l2(p22, p4) < 4e-2


def test_accumulation_with_regulariser_vs_autograd(cuda, tmp_path):
    """regulariser on: the accumulated gradient of two B = 2 micro-batches == the sum of their fp32 autograd gradients"""
    from test_fusion_orchestration import WordTokenizer
    base, ref_unet, clip = _base_dir(tmp_path)
    tok = WordTokenizer()
    delta = _delta(ref_unet, clip)
    tr = _trainer(base, tok, 0.05, False)
    tr.load_delta_state_dict(delta)
    mbs = _fixed(2)
    losses = [_step(tr, mb, accumulate=k > 0).item() for k, mb in enumerate(mbs)]
    torch.cuda.synchronize()
    ref_losses, g_rows, t_leaves, u_leaves = autograd_reference(
        tr, clip, ref_unet, delta, tok,
        [(mb['prompts'], mb['images'], mb['noise'], mb['timesteps'], mb['masks']) for mb in mbs], 0.05, False)
    res = group_errors(tr, g_rows, t_leaves, u_leaves)
    print(f'accumulated 2 x B=2 with the regulariser: losses {["%.5f" % x for x in losses]} vs autograd '
          f'{["%.5f" % x for x in ref_losses]};  ' + format_errors(res))
    for x, y in zip(losses, ref_losses):
        assert abs(x - y) < 2e-2 * abs(y)
    for name, (r, c, _) in res.items():
        assert r < 4e-2 and c > 0.998, name


class _FixedNoise:
    """the trainer with each call's noise and timesteps taken from the micro-batch, so that train() can be held to a
    deterministic target; records the `accumulate` of every call"""

    def __init__(self, tr):
        self.tr, self.calls = tr, []

    @property
    def engine(self):
        return self.tr.engine

    def refresh(self):
        self.tr.refresh()

    def __call__(self, images, prompts, masks, img_masks, accumulate=False):
        mb = next(m for m in self.batches if m['images'] is images)
        self.calls.append(accumulate)
        return self.tr(images, prompts, masks, img_masks, noise=mb['noise'], timesteps=mb['timesteps'],
                       accumulate=accumulate)


def test_train_loop_gradient_accumulation(cuda, tmp_path, monkeypatch):
    """train(..., batch_size_per_gpu=2, gradient_accumulation_steps=2) over 8 samples: 4 micro-batches, `accumulate` on
    every second, 2 optimiser steps; the gradient each step applies (grads x grad_scale) is the B = 4 gradient of its four
    samples, and the learning rates follow the linear schedule advanced per micro-step (lr at micro-steps 1 and 3 of 4)"""
    from test_fusion_orchestration import WordTokenizer
    import train_edlora as te
    base, ref_unet, clip = _base_dir(tmp_path)
    delta = _delta(ref_unet, clip)
    one, tr = _trainer(base, WordTokenizer(), None, False), _trainer(base, WordTokenizer(), None, False)
    for x in (one, tr):
        x.load_delta_state_dict(delta)
    (b4,) = _fixed(1)
    _step(one, b4)
    g4 = one.state.grads[:one.state.n].cpu().clone()
    del one
    wrapped = _FixedNoise(tr)
    wrapped.batches = _fixed(2) + _fixed(2, seed=61)
    seen = []
    real_step = te.optimizer_step

    def recording_step(state, grad_scale, norm_out=None):
        seen.append((state.grads[:state.n].cpu() * grad_scale, tuple(state.lrs)))
        real_step(state, grad_scale, norm_out=norm_out)

    monkeypatch.setattr(te, 'optimizer_step', recording_step)
    losses = te.train(wrapped, wrapped.batches, dataset_len=8, batch_size_per_gpu=2, gradient_accumulation_steps=2,
                      emb_norm_threshold=10.0)           # no freeze of the rows: every group keeps its schedule
    assert te.total_iterations(8, 2, 1, 2) == 2 and len(losses) == 2 and len(seen) == 2
    assert wrapped.calls == [False, True, False, True]
    res, (e, c) = _compare_flat(tr.state, seen[0][0], g4)
    print(f'train() with gradient_accumulation_steps=2, first step vs B=4: flat rel-L2 {e:.3e} cos {c:.5f};  '
          + format_errors(res) + f';  lrs {seen[0][1]} then {seen[1][1]}')
    assert e < 4e-2
    base_lrs = tuple(float(FINETUNE[k]['lr']) for k in ('text_embedding', 'text_encoder', 'unet'))
    for (_, lrs), k in zip(seen, (1, 3)):
        assert lrs == pytest.approx([te.linear_lr(b, k, 4) for b in base_lrs], rel=1e-12)


# ------------------------------------------------------------------------------------------------ c. launch audits
@pytest.mark.parametrize('B', [4, 1], ids=lambda b: f'B{b}')
def test_launch_audits_train_sd15_full(cuda, B):
    """every GEMM, attention and norm / elementwise launch of the full-size training step and its optimiser step at batch
    B passes its float64 bound and write window (one engine, one step and one optimiser step per recorder)"""
    import attention_audit as aa
    import gemm_audit as ga
    import norm_audit as na
    w = walks.build_train_sd15_full(use_graph=False, B=B)
    stats = {}
    for name, mod in (('gemm', ga), ('attention', aa), ('norm', na)):
        st = mod.Stats()
        walks.train_sd15_full(lambda: mod.Recorder(st), w=w)
        stats[name] = st
        print(f'\n{name} launch audit, full-size training step at B = {B}:\n' + st.table())
    del w
    torch.cuda.empty_cache()
    for name, st in stats.items():
        assert not st.failures, f'{name}: ' + '\n'.join(st.failures[:20])
        assert st.rows, name


# ------------------------------------------------------------------------------------------------ d. train_edlora.py -opt
@pytest.mark.parametrize('bs,accum', [(4, 1), (2, 2)], ids=['batch4', 'batch2_accum2'])
def test_train_edlora_opt_batch(cuda, tmp_path, bs, accum):
    """`train_edlora.py -opt` on the synthetic model directory over 8 samples: finite losses, total_iterations optimiser
    steps, a checkpoint with the reference's keys and shapes (16 x 768 rows per concept word, rank-4 CLIPAttention and
    Attention LoRA pairs on every projection)"""
    from mixofshow.utils import model_io
    from synth import make_pretrained_dir
    from test_e2e_flows_gpu import _train_one
    base = make_pretrained_dir(str(tmp_path / 'base'))
    ckpt = _train_one(tmp_path, base, 'cat', '<cat1>+<cat2>', '<rand-0.013>+a', 'photo of a <TOK>', seed=1,
                      batch_size_per_gpu=bs, gradient_accumulation_steps=accum)
    params = torch.load(ckpt)['params']
    usd = model_io.load_unet(base).state_dict()
    want = {k[:-len('.weight')] for k in usd
            if k.endswith('.weight') and ('.attn1.' in k or '.attn2.' in k) and 'norm' not in k}
    got = {k.rsplit('.lora_', 1)[0] for k in params['unet']}
    assert got == want and len(params['unet']) == 2 * len(want)
    for m in want:
        W = usd[m + '.weight']
        assert tuple(params['unet'][m + '.lora_down.weight'].shape) == (4, W.shape[1])
        assert tuple(params['unet'][m + '.lora_up.weight'].shape) == (W.shape[0], 4)
    for k, v in params['text_encoder'].items():
        assert '.self_attn.' in k and tuple(v.shape) in ((4, 768), (768, 4)), (k, tuple(v.shape))
    print(f'train_edlora.py -opt batch {bs} x accumulation {accum}: {json.dumps(sorted(params))}, '
          f'{len(params["unet"])} unet / {len(params["text_encoder"])} text tensors')
