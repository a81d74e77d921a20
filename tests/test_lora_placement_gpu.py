"""Whole-block LoRA placements on the GPU: `where: Transformer2DModel` (UNet) and `where: CLIPEncoderLayer` (text encoder),
trainer_edlora.py:100-133.  Besides the attention projections these put a LoRA on proj_in / proj_out (1x1 convs),
ff.net.0.proj (GEGLU, C -> 8C) and ff.net.2 of every transformer block, and on mlp.fc1 / mlp.fc2 of every CLIP layer.

  * mos_lora_grad at every shape these modules have at SD1.5 sizes, against float64 (the GEGLU projection of the
    1280-channel blocks, K = 1280 / N = 10240, no longer fits the shared-memory staging and reads D / U from global memory);
  * the full trainer step (text encoder + UNet) against fp32 autograd for the three non-default placement combinations,
    per parameter group and per module kind, and a UNet step at the SD1.5 channel widths;
  * checkpoints (reference key sets and shapes, bit-exact round trip, CLIP pads stay zero under AdamW), the train loop,
    and sampling with a whole-block LoRA (un-merged vs the fp32 oracle / transformers, and vs merged weights).

Every bound has the worst value measured on an H100 80GB HBM3 next to it."""
import json

import pytest
import torch

from gpu_helpers import canary, rel_l2_64, same_bits, untouched, window_mask
from test_trainer_full_gpu import FINETUNE, _base_dir, _cos, rel_l2

pytestmark = pytest.mark.gpu

# (label, K, N, tokens per sample): the LoRA'd GEMMs of the new placements at SD1.5 sizes, 64 x 64 latents
# (UNet: tokens = H*W of the block's level; CLIP: 16 layer-wise prompts of 77 tokens per sample, padded as clip_engine)
WIDE_SHAPES = [
    ('ff1_320', 320, 2560, 4096), ('ff1_640', 640, 5120, 1024), ('ff1_1280', 1280, 10240, 256),
    ('ff2_320', 1280, 320, 4096), ('ff2_640', 2560, 640, 1024), ('ff2_1280', 5120, 1280, 256),
    ('proj_320', 320, 320, 4096), ('proj_640', 640, 640, 1024), ('proj_1280', 1280, 1280, 256),
    ('proj_mid', 1280, 1280, 64), ('clip_fc1', 768, 3200, 16 * 77), ('clip_fc2', 3200, 800, 16 * 77),
]


def _lora_grad_ref(x, dy, D, U, alpha):
    x, dy, D, U = x.double(), dy.double(), D.double(), U.double()
    return alpha * (dy @ U).t() @ x, alpha * dy.t() @ (x @ D.t())


@pytest.mark.parametrize('B', [1, 8])
@pytest.mark.parametrize('label,K,N,T', WIDE_SHAPES, ids=[s[0] for s in WIDE_SHAPES])
def test_lora_grad_wide_shapes(cuda, label, K, N, T, B):
    from mos_b200 import ops
    M = B * T
    g = torch.Generator().manual_seed(K + N + B)
    x = torch.randn(M, K, generator=g).to(torch.bfloat16).to(cuda)
    dy = (torch.randn(M, N, generator=g) * 0.1).to(torch.bfloat16).to(cuda)
    D = (torch.rand(4, K, generator=g) * 2 - 1).div(K ** 0.5).to(cuda)
    U = (torch.randn(N, 4, generator=g) * 0.05).to(cuda)
    alpha = 0.7
    ws = torch.empty(128 * 4 * (K + N), device=cuda)
    dd, du = canary((4 + 2, K), cuda, torch.float32), canary((N + 3, 4), cuda, torch.float32)
    ops.lora_grad(x, dy, D, U, alpha, ws, dd[:4], du[:N], M=M, K=K, N=N)
    torch.cuda.synchronize()
    rD, rU = _lora_grad_ref(x, dy, D, U, alpha)
    eD, eU = rel_l2_64(dd[:4], rD), rel_l2_64(du[:N], rU)
    print(f'{label} M={M}: dD rel-L2 {eD:.2e}, dU rel-L2 {eU:.2e}')
    assert eD < 1e-5 and eU < 1e-5                                  # measured <= 9.3e-7 (fp32 accumulation)
    assert untouched(dd, window_mask(dd, slice(0, 4))) and untouched(du, window_mask(du, slice(0, N)))
    # bitwise repeatable; accumulate=1 adds onto what is there (one fused multiply-add per element)
    d2, u2 = torch.empty(4, K, device=cuda), torch.empty(N, 4, device=cuda)
    ops.lora_grad(x, dy, D, U, alpha, ws, d2, u2, M=M, K=K, N=N)
    assert same_bits(d2, dd[:4]) and same_bits(u2, du[:N])
    base_d, base_u = torch.randn(4, K, generator=g).to(cuda), torch.randn(N, 4, generator=g).to(cuda)
    d3, u3 = base_d.clone(), base_u.clone()
    ops.lora_grad(x, dy, D, U, alpha, ws, d3, u3, M=M, K=K, N=N, accumulate=True)
    eaD, eaU = rel_l2_64(d3, base_d.double() + rD), rel_l2_64(u3, base_u.double() + rU)
    assert eaD < 1e-5 and eaU < 1e-5                                # measured <= 9.3e-7 as well


def _combo(text_where, unet_where):
    cfg = json.loads(json.dumps(FINETUNE))
    cfg['text_encoder']['lora_cfg']['where'] = text_where
    cfg['unet']['lora_cfg']['where'] = unet_where
    return cfg


def _kind(m):
    for k in ('proj_in', 'proj_out', 'ff.net.0.proj', 'ff.net.2', 'mlp.fc1', 'mlp.fc2'):
        if m.endswith(k):
            return k
    return 'attention'


COMBOS = [('CLIPEncoderLayer', 'Attention'), ('CLIPAttention', 'Transformer2DModel'),
          ('CLIPEncoderLayer', 'Transformer2DModel')]


@pytest.mark.parametrize('text_where,unet_where', COMBOS)
def test_full_trainer_step_placements_vs_autograd(cuda, tmp_path, text_where, unet_where):
    """The attention regulariser is off here: it divides by the maximum of the concept-token attention over the batch, and
    its gradient jumps between elements that lie within bf16 rounding of that maximum.  With it on, the
    CLIPAttention / Transformer2DModel case puts every group 3-8e-2 away from autograd (the same for repeated runs), while
    the loss agrees to 0.02 % and the same step without the regulariser agrees to 1.4e-2.  The regulariser itself is
    covered by test_trainer_full_gpu and test_attn_reg_gpu, and by the train loop below."""
    from test_fusion_orchestration import WordTokenizer
    from mixofshow.pipelines.pipeline_edlora import bind_concept_prompt
    from mixofshow.pipelines.trainer_edlora import EDLoRATrainer
    from mixofshow.utils.ptp_util import AttentionStore
    from oracle import inject, train_ref
    from oracle.schedulers import DDPMScheduler
    base, ref_unet, clip = _base_dir(tmp_path)
    tok = WordTokenizer()
    reg_w = None
    tr = EDLoRATrainer(base, '<c1>+<c2>', '<rand-0.02>+<rand-0.02>', True, finetune_cfg=_combo(text_where, unet_where),
                       attn_reg_weight=reg_w, reg_full_identity=False, tokenizer=tok, latent_size=(16, 16))
    ids_concept = tr.get_all_concept_token_ids()
    g = torch.Generator().manual_seed(5)
    delta = {'new_concept_embedding': {'<c1>': torch.randn(16, 768, generator=g) * 0.02,
                                       '<c2>': torch.randn(16, 768, generator=g) * 0.02},
             'text_encoder': inject.random_lora_state(clip, seed=3, where=text_where, up_std=0.05),
             'unet': inject.random_lora_state(ref_unet, seed=10, where=unet_where)}
    tr.load_delta_state_dict(delta)
    B, H = 2, 16
    prompts = ['photo of a <c1> <c2>', 'the <c1> <c2> on a beach']
    lat, noise = torch.randn(B, 4, H, H, generator=g), torch.randn(B, 4, H, H, generator=g)
    t = torch.tensor([130, 811])
    masks = (torch.rand(B, 1, H, H, generator=g) > 0.5).float()
    masks[:, :, 4:9, 4:9] = 1.0
    masks[:, :, 0, 0] = 0.0
    loss = tr(lat, prompts, masks, torch.ones_like(masks), noise=noise, timesteps=t)
    torch.cuda.synchronize()
    clip.resize_token_embeddings(49408 + 32)
    emb = clip.get_input_embeddings().weight
    with torch.no_grad():
        emb[49408:49408 + 16] = delta['new_concept_embedding']['<c1>']
        emb[49408 + 16:49408 + 32] = delta['new_concept_embedding']['<c2>']
    emb.requires_grad_(True)
    t_leaves = {k: v.clone().requires_grad_(True) for k, v in delta['text_encoder'].items()}
    u_leaves = {k: v.clone().requires_grad_(True) for k, v in delta['unet'].items()}
    inject.inject_lora(clip, t_leaves, 1.0)
    inject.inject_lora(ref_unet, u_leaves, 1.0)
    ctl = AttentionStore(training=True)
    inject.install_control_processors(ref_unet, ctl)
    ids = tok(bind_concept_prompt(prompts, tr.new_concept_cfg), padding='max_length', max_length=77,
              return_tensors='pt').input_ids
    ehs = clip(ids)[0].view(B, 16, 77, 768)
    pos = train_ref.concept_token_positions(ids, B, ids_concept)
    noisy = DDPMScheduler().add_noise(lat, noise, t)
    loss_ref, _, _ = train_ref.train_loss(ref_unet, ctl, noisy, t, ehs, noise, masks, masks, pos, reg_full_identity=False,
                                          attn_reg_weight=reg_w)
    loss_ref.backward()
    print(f'[{text_where} / {unet_where}] loss {loss.item():.6f} vs autograd {loss_ref.item():.6f}')
    assert abs(loss.item() - loss_ref.item()) < 2e-2 * abs(loss_ref.item())       # measured 0.03 %
    g_emb_ref = emb.grad[49408:49408 + 32]
    e0, c0 = rel_l2(tr.text_engine.emb_grad, g_emb_ref), _cos(tr.text_engine.emb_grad, g_emb_ref)
    print(f'  embedding rows: rel-L2 {e0:.3e} cos {c0:.5f}')
    assert e0 < 4e-2 and c0 > 0.998                                  # measured 9.3e-3, cos 0.99996
    for name, eng, leaves in (('text', tr.text_engine, t_leaves), ('unet', tr.engine, u_leaves)):
        assert sorted(f'{m}.lora_{p}.weight' for m in eng.lora_grad_dict() for p in ('down', 'up')) == sorted(leaves)
        groups = {}
        for m, (gd, gu) in eng.lora_grad_dict().items():
            for k in ('all', _kind(m)):
                fg, fr = groups.setdefault(k, ([], []))
                fg += [gd.flatten().cpu(), gu.flatten().cpu()]
                fr += [leaves[m + '.lora_down.weight'].grad.reshape(gd.shape).flatten(),
                       leaves[m + '.lora_up.weight'].grad.reshape(gu.shape).flatten()]
        for k, (fg, fr) in groups.items():
            fg, fr = torch.cat(fg), torch.cat(fr)
            e, c = rel_l2(fg, fr), _cos(fg, fr)
            print(f'  {name} LoRA {k} ({fg.numel()}): rel-L2 {e:.3e} cos {c:.5f}')
            assert e < 4e-2 and c > 0.998               # measured worst: rel-L2 1.4e-2, cos 0.99991 (ff.net.2)
        kinds = set(groups) - {'all', 'attention'}
        want = {'text': {'mlp.fc1', 'mlp.fc2'} if text_where == 'CLIPEncoderLayer' else set(),
                'unet': {'proj_in', 'proj_out', 'ff.net.0.proj', 'ff.net.2'} if unet_where == 'Transformer2DModel'
                else set()}[name]
        assert kinds == want


def test_unet_step_sd15_channels_transformer2d(cuda):
    """The UNet side at the SD1.5 channel widths (320, 640, 1280, 1280; one layer per block to stay small) with
    `where: Transformer2DModel`: ff.net.0.proj reaches N = 10240 (the global-memory lora_grad path).  fp32 oracle on the
    GPU, autograd."""
    from mixofshow.utils.ptp_util import AttentionStore
    from mos_b200.engine import ehs_to_layer_major
    from mos_b200.train_engine import TrainEngine
    from oracle import inject, train_ref
    from oracle import unet as ou
    from oracle.schedulers import DDPMScheduler
    cfg = dict(block_out_channels=(320, 640, 1280, 1280), layers_per_block=1)
    ref = ou.build_unet(0, cfg)
    lora = inject.random_lora_state(ref, seed=10, where='Transformer2DModel')
    sd = {k: v.detach().clone() for k, v in ref.state_dict().items()}
    ref = ref.cuda()
    leaves = {k: v.clone().cuda().requires_grad_(True) for k, v in lora.items()}
    inject.inject_lora(ref, leaves, 1.0)
    ctl = AttentionStore(training=True)
    n_x = inject.install_control_processors(ref, ctl)
    g = torch.Generator().manual_seed(5)
    B, H = 2, 16
    x0, noise = torch.randn(B, 4, H, H, generator=g), torch.randn(B, 4, H, H, generator=g)
    t = torch.tensor([77, 640])
    ehs = torch.randn(B, n_x, 77, 768, generator=g).to(torch.bfloat16).float()
    masks = torch.ones(B, 1, H, H)
    noisy = DDPMScheduler().add_noise(x0, noise, t)
    loss_ref, _, _ = train_ref.train_loss(ref, ctl, noisy.cuda(), t.cuda(), ehs.cuda(), noise.cuda(), masks.cuda(),
                                          masks.cuda(), None, reg_full_identity=True, attn_reg_weight=None)
    loss_ref.backward()
    eng = TrainEngine(sd, B, H, H, lora=lora, attn_reg_weight=None, where='Transformer2DModel',
                      block_out=cfg['block_out_channels'], layers=1)
    assert max(N for (_, _, _, _, _, N) in eng.lora_views.values()) == 10240
    out = eng.forward_backward(x0.cuda(), noise.cuda(), t.cuda(), ehs_to_layer_major(ehs.cuda(), n_x), masks.cuda())
    torch.cuda.synchronize()
    print(f'SD1.5 channels, Transformer2DModel: loss {out[0].item():.6f} vs autograd {loss_ref.item():.6f}')
    assert abs(out[0].item() - loss_ref.item()) < 2e-2 * abs(loss_ref.item())
    groups = {}
    for m, (gd, gu) in eng.lora_grad_dict().items():
        for k in ('all', _kind(m)):
            fg, fr = groups.setdefault(k, ([], []))
            fg += [gd.flatten().cpu(), gu.flatten().cpu()]
            fr += [leaves[m + '.lora_down.weight'].grad.reshape(gd.shape).flatten().cpu(),
                   leaves[m + '.lora_up.weight'].grad.reshape(gu.shape).flatten().cpu()]
    for k, (fg, fr) in groups.items():
        fg, fr = torch.cat(fg), torch.cat(fr)
        e, c = rel_l2(fg, fr), _cos(fg, fr)
        print(f'  {k} ({fg.numel()}): rel-L2 {e:.3e} cos {c:.5f}')
        assert e < 4e-2 and c > 0.998                   # measured worst: rel-L2 2.5e-2, cos 0.99970 (ff.net.0.proj)


def test_checkpoints_whole_block(cuda, tmp_path):
    """Reference key sets and shapes (4-D for the 1x1 convs), a bit-exact load -> save round trip, and CLIP pads that
    stay exactly zero after optimiser steps."""
    from test_fusion_orchestration import WordTokenizer
    from mixofshow.pipelines.trainer_edlora import EDLoRATrainer
    from mos_b200.dp import optimizer_step
    from oracle import inject
    base, ref_unet, clip = _base_dir(tmp_path, clip_layers=1)
    tr = EDLoRATrainer(base, '<c1>+<c2>', '<rand-0.02>+<rand-0.02>', True,
                       finetune_cfg=_combo('CLIPEncoderLayer', 'Transformer2DModel'), attn_reg_weight=0.01,
                       reg_full_identity=False, tokenizer=WordTokenizer(), latent_size=(16, 16))
    g = torch.Generator().manual_seed(2)
    m = torch.zeros(2, 1, 16, 16)
    m[:, :, 3:12, 4:13] = 1
    args = (torch.randn(2, 4, 16, 16, generator=g), ['photo of a <c1> <c2>', 'a <c1> <c2> smiling'], m,
            torch.ones(2, 1, 16, 16))
    tr(*args)                                               # builds the engines (fresh LoRALinearLayer init)
    d0 = tr.delta_state_dict()
    want_u = inject.random_lora_state(ref_unet, where='Transformer2DModel')
    want_t = inject.random_lora_state(clip, where='CLIPEncoderLayer')
    for got, want in ((d0['unet'], want_u), (d0['text_encoder'], want_t)):
        assert set(got) == set(want)
        for k in want:
            assert tuple(got[k].shape) == tuple(want[k].shape), k
            if k.endswith('lora_up.weight'):
                assert torch.count_nonzero(got[k]) == 0, k      # up = 0 at init
            else:
                assert got[k].abs().max().item() <= 1.0 / want[k].shape[1] ** 0.5 + 1e-7
    assert d0['unet']['down_blocks.0.attentions.0.proj_in.lora_down.weight'].ndim == 4
    assert sum(v.numel() for v in d0['unet'].values()) == sum(v.numel() for v in want_u.values())
    # round trip
    src = {'new_concept_embedding': d0['new_concept_embedding'], 'unet': inject.random_lora_state(ref_unet, seed=4,
           where='Transformer2DModel'), 'text_encoder': inject.random_lora_state(clip, seed=5, where='CLIPEncoderLayer')}
    tr.load_delta_state_dict(src)
    d1 = tr.delta_state_dict()
    for part in ('unet', 'text_encoder'):
        for k, v in src[part].items():
            assert torch.equal(d1[part][k], v.float()), k
    # pads of the CLIP flat LoRA stay exactly zero through training steps
    te = tr.text_engine
    for _ in range(3):
        tr(*args)
        optimizer_step(tr.state, 1.0)
        tr.refresh()
    torch.cuda.synchronize()
    I = te.I
    for mname, (D, U, gD, gU, K, N) in te.lora_views.items():
        if mname.endswith('mlp.fc1'):
            assert torch.count_nonzero(U[I:]) == 0 and torch.count_nonzero(gU[I:]) == 0
            assert U[:I].abs().max().item() > 0
        elif mname.endswith('mlp.fc2'):
            assert torch.count_nonzero(D[:, I:]) == 0 and torch.count_nonzero(gD[:, I:]) == 0
    for i in range(te.n_layers):
        assert torch.count_nonzero(te.w[i]['fc1']['lora_up'][I:]) == 0
        assert torch.count_nonzero(te.w[i]['fc2']['lora_down'][:, I:]) == 0


def test_train_loop_whole_block(cuda, tmp_path):
    import train_edlora as tel
    from test_fusion_orchestration import WordTokenizer
    from mixofshow.pipelines.trainer_edlora import EDLoRATrainer
    base, _, _ = _base_dir(tmp_path, clip_layers=1)
    tr = EDLoRATrainer(base, '<c1>+<c2>', '<rand-0.013>+<rand-0.013>', True,
                       finetune_cfg=_combo('CLIPEncoderLayer', 'Transformer2DModel'), attn_reg_weight=0.01,
                       reg_full_identity=False, tokenizer=WordTokenizer(), latent_size=(16, 16))
    g = torch.Generator().manual_seed(1)
    m = torch.zeros(2, 1, 16, 16)
    m[:, :, 3:12, 4:13] = 1
    batch = {'images': torch.randn(2, 4, 16, 16, generator=g), 'prompts': ['photo of a <c1> <c2>', 'a <c1> <c2> smiling'],
             'masks': m, 'img_masks': torch.ones(2, 1, 16, 16)}
    tr(batch['images'], batch['prompts'], batch['masks'], batch['img_masks'])
    d0 = tr.delta_state_dict()
    losses = tel.train(tr, [batch] * 10, dataset_len=20, batch_size_per_gpu=2, print_freq=0)
    d1 = tr.delta_state_dict()
    print('    losses', ' '.join(f'{x:.4f}' for x in losses))
    for part, keys in (('unet', ('proj_in', 'proj_out', 'ff.net.0.proj', 'ff.net.2', 'attn1.to_q')),
                       ('text_encoder', ('mlp.fc1', 'mlp.fc2', 'q_proj'))):
        for kk in keys:
            moved = [k for k in d1[part] if f'{kk}.lora_up' in k and not torch.equal(d1[part][k], d0[part][k])]
            assert moved, (part, kk)
    assert not torch.equal(d1['new_concept_embedding']['<c1>'], d0['new_concept_embedding']['<c1>'])
    assert losses[-1] < losses[0]


def test_sampling_with_whole_block_lora(cuda):
    """Sampling engines with an un-merged whole-block LoRA: UNetEngine vs the fp32 oracle, CLIPTextEngine (fc1 / fc2
    LoRA) vs transformers, and the un-merged UNet vs merged weights (merge_lora_into_weight, as convert_edlora)."""
    from transformers import CLIPTextConfig, CLIPTextModel
    from mixofshow.utils.convert_edlora_to_diffusers import merge_lora_into_weight
    from mos_b200.clip_engine import CLIPTextEngine
    from mos_b200.engine import UNetEngine, ehs_to_layer_major
    from oracle import inject
    from oracle import unet as ou
    unet = ou.build_unet(0, ou.TINY)
    inject.install_edlora_processors(unet)
    lora = inject.random_lora_state(unet, seed=10, where='Transformer2DModel', up_std=0.05)
    sd = {k: v.clone() for k, v in unet.state_dict().items()}
    inject.inject_lora(unet, lora, 0.8)
    g = torch.Generator().manual_seed(1)
    B, H = 2, 32
    lat = torch.randn(B, 4, H, H, generator=g)
    ehs = torch.randn(B, 16, 77, 768, generator=g)
    tt = torch.tensor([501.0, 501.0])
    with torch.no_grad():
        ref = unet(lat, tt, ehs).sample
    kw = dict(block_out=ou.TINY['block_out_channels'], layers=ou.TINY['layers_per_block'])
    eng = UNetEngine(sd, B, H, H, lora=lora, lora_alpha=0.8, **kw)
    nx = len(eng.xattn_names)
    eps = eng.forward(lat.cuda(), tt.cuda(), ehs_to_layer_major(ehs[:, :nx].cuda(), nx)).clone()
    base = UNetEngine(sd, B, H, H, **kw).forward(lat.cuda(), tt.cuda(), ehs_to_layer_major(ehs[:, :nx].cuda(), nx)).clone()
    merged_sd = merge_lora_into_weight(sd, lora, 'unet', 0.8)
    eps_m = UNetEngine(merged_sd, B, H, H, **kw).forward(lat.cuda(), tt.cuda(),
                                                         ehs_to_layer_major(ehs[:, :nx].cuda(), nx)).clone()
    torch.cuda.synchronize()
    e, e_base, e_m = rel_l2(eps, ref), rel_l2(base, ref), rel_l2(eps, eps_m)
    print(f'UNet whole-block LoRA: rel-L2 {e:.3e} (without the LoRA {e_base:.3e}); un-merged vs merged {e_m:.3e}')
    assert e < 5e-3 and e_base > 2 * e                       # measured 1.1e-3; bound of the fp16 forward tests
    assert e_m < 5e-3                                          # measured 1.1e-3
    cfg = CLIPTextConfig(vocab_size=49408, hidden_size=768, intermediate_size=3072, num_hidden_layers=2,
                         num_attention_heads=12, max_position_embeddings=77)
    torch.manual_seed(0)
    model = CLIPTextModel(cfg).eval()
    csd = {k: v.clone() for k, v in model.state_dict().items()}
    tlora = inject.random_lora_state(model, seed=7, where='CLIPEncoderLayer', up_std=0.05)
    ids = torch.randint(0, 49407, (16, 77), generator=g)
    ids[:, 0] = 49406
    ids[:, 9:] = 49407
    inject.inject_lora(model, tlora, 0.8)
    with torch.no_grad():
        cref = model(ids)[0]
    out = CLIPTextEngine(csd, 16, lora=tlora, lora_alpha=0.8)(ids)
    attn_only = {k: v for k, v in tlora.items() if '.mlp.' not in k}
    out_a = CLIPTextEngine(csd, 16, lora=attn_only, lora_alpha=0.8)(ids)
    out_m = CLIPTextEngine(csd, 16, lora=tlora, lora_alpha=0.8, merge_lora=True)(ids)
    torch.cuda.synchronize()
    ec, ea, em = rel_l2(out, cref), rel_l2(out_a, cref), rel_l2(out_m, cref)
    print(f'CLIP fc1/fc2 LoRA: rel-L2 {ec:.3e} (attention LoRA only {ea:.3e}, merged {em:.3e})')
    assert ec < 2e-2 and em < 2e-2 and ea > 2 * ec             # measured 6.1e-3 / 6.2e-3; bound of test_clip_gpu
