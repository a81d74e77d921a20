"""EDLoRATrainer with every non-empty subset of ED-LoRA's three parameter groups on the GPU (trainer_edlora.py:70-142).

For each combination: the captured step's loss and the gradients of every trained group against fp32 autograd through
transformers' CLIPTextModel chained into the oracle UNet with `requires_grad` on the same groups (tolerances of
test_trainer_full_gpu.py: rel-L2 <= 4e-2, cosine >= 0.998, loss within 2 %, widened for a group only as far as twice the
error that bf16 autocast alone puts into the same autograd run on the same batch); the launches of absent work are not
issued (counted through the ops.* wrappers while the step is captured and while train() runs, each LoRA-gradient launch
attributed to its network by where it writes in the flat gradient); after a few optimiser steps of
train() every untrained tensor is bit-identical to its initial value.  The new launch sequences (frozen UNet, CLIP
without LoRA, CLIP with constant rows, a forward-only text encoder) are audited against their float64 references and
write windows, and `train_edlora.py -opt` trains and validates a config with the text-encoder group switched off."""
import collections

import pytest
import torch
import yaml

from test_finetune_groups import COMBOS, combo_id, finetune_cfg
from test_trainer_full_gpu import _base_dir, _cos, rel_l2

pytestmark = pytest.mark.gpu

PROMPTS = ['photo of a <c1> <c2>', 'the <c1> <c2> on a beach']
COUNTED = ('lora_grad', 'lora_pack', 'clip_embed_bwd', 'quick_gelu_bwd', 'attention_bwd', 'gemm', 'splitk_finalize',
           'flat_adamw_step')
OUT_ARG = {'gemm': 2, 'splitk_finalize': 4}          # positional index of the output tensor


class LaunchCounter:
    """counts calls of the ops.* wrappers named in COUNTED (each is one library entry point) while active"""

    def __init__(self, monkeypatch):
        from mos_b200 import ops
        self.n = collections.Counter()
        self.outs = []
        self.lora_grad_dst = []              # d_down of every lora_grad launch: where in the flat gradient it writes
        self.lora_pack_tables = []           # the pointer table of every lora_pack launch: whose LoRA set it re-packs
        for name in COUNTED:
            fn = getattr(ops, name)

            def counted(*a, _fn=fn, _name=name, **k):
                self.n[_name] += 1
                if _name == 'lora_grad':
                    self.lora_grad_dst.append(a[6].data_ptr())
                if _name == 'lora_pack':
                    self.lora_pack_tables.append(a[0].data_ptr())
                if _name in OUT_ARG:
                    self.outs.append(a[OUT_ARG[_name]] if len(a) > OUT_ARG[_name] else k.get('out'))
                return _fn(*a, **k)
            monkeypatch.setattr(ops, name, counted)


def _trainer(base, combo, tok=None):
    from test_fusion_orchestration import WordTokenizer
    from mixofshow.pipelines.trainer_edlora import EDLoRATrainer
    return EDLoRATrainer(base, '<c1>+<c2>', '<rand-0.02>+<rand-0.02>', True, finetune_cfg=finetune_cfg(*combo),
                         attn_reg_weight=0.05, reg_full_identity=False, use_mask_loss=True,
                         tokenizer=tok or WordTokenizer(), latent_size=(16, 16))


def _data(ref_unet, clip, combo):
    """the checkpoint and batch of test_trainer_full_gpu.py's three-group step, drawn in the same order: the concept rows
    always, a random LoRA (non-zero up) for the LoRA groups that train -> (delta, latents, noise, timesteps, masks)"""
    from oracle import inject
    g = torch.Generator().manual_seed(5)
    d = {'new_concept_embedding': {c: torch.randn(16, 768, generator=g) * 0.02 for c in ('<c1>', '<c2>')},
         'text_encoder': {}, 'unet': {}}
    if combo[1]:
        d['text_encoder'] = inject.random_lora_state(clip, seed=3, where='CLIPAttention', up_std=0.05)
    if combo[2]:
        d['unet'] = inject.random_lora_state(ref_unet, seed=10)
    B, H = 2, 16
    lat, noise = torch.randn(B, 4, H, H, generator=g), torch.randn(B, 4, H, H, generator=g)
    masks = (torch.rand(B, 1, H, H, generator=g) > 0.5).float()
    masks[:, :, 4:9, 4:9] = 1.0
    masks[:, :, 0, 0] = 0.0
    return d, lat, noise, torch.tensor([130, 811]), masks


def _expected_absent(tr, counter, combo):
    emb, text, unet = combo
    n = counter.n
    if not unet:
        assert tr.engine.lora_views == {} and tr.engine.lora_table.numel() == 0
        assert not any('lora_down' in e for e in tr.engine.wb.values() if isinstance(e, dict))
    if not (emb or text):                        # no CLIP backward, no d(text embeddings), no text K / V dX GEMMs
        assert tr.engine.d_ehs is None and not hasattr(tr.text_engine, 'backward')
        assert not any(k.endswith('attn2.to_k') or k.endswith('attn2.to_v') for k in tr.engine.wb)
        assert n['quick_gelu_bwd'] == 0 and n['clip_embed_bwd'] == 0
    else:
        assert n['quick_gelu_bwd'] > 0
        d = tr.engine.d_ehs
        assert sum(1 for o in counter.outs if o is not None and o.data_ptr() == d.data_ptr()) > 0
    # every LoRA-gradient launch writes into the flat-gradient range of a trained LoRA group; a frozen network issues none
    st = tr.state
    ge = st.group_end
    owner = collections.Counter()
    for ptr in counter.lora_grad_dst:
        off = (ptr - st.grads.data_ptr()) // st.grads.element_size()
        owner['text' if ge[0] <= off < ge[1] else 'unet' if ge[1] <= off < ge[2] else 'outside'] += 1
    assert owner['outside'] == 0, owner
    assert (owner['text'] > 0) == text and (owner['unet'] > 0) == unet, owner
    assert n['lora_grad'] == owner['text'] + owner['unet']
    if not emb:
        assert n['clip_embed_bwd'] == 0
    else:
        assert n['clip_embed_bwd'] > 0


@pytest.mark.parametrize('combo', COMBOS, ids=combo_id)
def test_step_vs_autograd(cuda, tmp_path, monkeypatch, combo):
    from test_fusion_orchestration import WordTokenizer
    from mixofshow.pipelines.pipeline_edlora import bind_concept_prompt
    from mixofshow.utils.ptp_util import AttentionStore
    from oracle import inject, train_ref
    from oracle.schedulers import DDPMScheduler
    emb_on, text_on, unet_on = combo
    base, ref_unet, clip = _base_dir(tmp_path)
    tok = WordTokenizer()
    tr = _trainer(base, combo, tok)
    delta, lat, noise, t, masks = _data(ref_unet, clip, combo)
    tr.load_delta_state_dict(delta)
    counter = LaunchCounter(monkeypatch)
    loss = tr(lat, PROMPTS, masks, torch.ones_like(masks), noise=noise, timesteps=t)    # warm-up + capture + replay
    torch.cuda.synchronize()
    monkeypatch.undo()
    _expected_absent(tr, counter, combo)
    # ---------------- autograd with requires_grad on the same groups: fp32, and bf16 autocast for the noise floor
    ids_concept = tr.get_all_concept_token_ids()
    clip.resize_token_embeddings(49408 + 32)
    emb = clip.get_input_embeddings().weight
    with torch.no_grad():
        emb[49408:49408 + 16] = delta['new_concept_embedding']['<c1>']
        emb[49408 + 16:49408 + 32] = delta['new_concept_embedding']['<c2>']
    for p in list(clip.parameters()) + list(ref_unet.parameters()):
        p.requires_grad_(False)
    emb.requires_grad_(emb_on)
    t_leaves = {k: v.clone().requires_grad_(True) for k, v in delta['text_encoder'].items()}
    u_leaves = {k: v.clone().requires_grad_(True) for k, v in delta['unet'].items()}
    if t_leaves:
        inject.inject_lora(clip, t_leaves, 1.0)
    if u_leaves:
        inject.inject_lora(ref_unet, u_leaves, 1.0)
    ids = tok(bind_concept_prompt(PROMPTS, tr.new_concept_cfg), padding='max_length', max_length=77,
              return_tensors='pt').input_ids
    pos = train_ref.concept_token_positions(ids, 2, ids_concept)
    noisy = DDPMScheduler().add_noise(lat, noise, t)
    # the engines' gradients, flattened per group in the engines' module order
    ours, order = {}, {}
    if emb_on:
        ours['rows'] = tr.text_engine.emb_grad.flatten().cpu()
    for name, on, eng in (('text', text_on, tr.text_engine), ('unet', unet_on, tr.engine)):
        if on:
            grads = eng.lora_grad_dict()
            order[name] = [(m, gd.shape, gu.shape) for m, (gd, gu) in grads.items()]
            ours[name] = torch.cat([x.flatten().cpu() for gd, gu in grads.values() for x in (gd, gu)])

    def autograd(bf16):
        for p in [emb, *t_leaves.values(), *u_leaves.values()]:
            p.grad = None
        ctl = AttentionStore(training=True)
        inject.install_control_processors(ref_unet, ctl)
        with torch.autocast('cpu', dtype=torch.bfloat16, enabled=bf16):
            ehs = clip(ids)[0].view(2, 16, 77, 768)
            loss_r, _, _ = train_ref.train_loss(ref_unet, ctl, noisy, t, ehs, noise, masks, masks, pos,
                                                reg_full_identity=False, attn_reg_weight=0.05)
        loss_r.float().backward()
        out = {}
        if emb_on:
            out['rows'] = emb.grad[49408:49408 + 32].float().flatten().clone()
        for name, leaves in (('text', t_leaves), ('unet', u_leaves)):
            if name in order:
                out[name] = torch.cat([leaves[m + f'.lora_{s}.weight'].grad.float().reshape(shp).flatten()
                                       for m, sd, su in order[name] for s, shp in (('down', sd), ('up', su))])
        return loss_r.item(), out

    loss_bf, g_bf = autograd(True)
    loss_ref, g_ref = autograd(False)
    msg = [f'{combo_id(combo)}: loss {loss.item():.6f} vs {loss_ref:.6f}']
    assert abs(loss.item() - loss_ref) < 2e-2 * abs(loss_ref)
    for name, g in ours.items():
        r, c = rel_l2(g, g_ref[name]), _cos(g, g_ref[name])
        r_bf, c_bf = rel_l2(g_bf[name], g_ref[name]), _cos(g_bf[name], g_ref[name])
        msg.append(f'{name}: rel-L2 {r:.3e} cos {c:.5f} (bf16 autocast autograd: {r_bf:.3e} / {c_bf:.5f})')
        assert r < max(4e-2, 2 * r_bf) and c > min(0.998, 1 - 2 * (1 - c_bf)), msg[-1]
    assert tr.state.grads.numel() == sum(tr.flat_group_sizes()) + 2      # the one all-reduce: present groups + 2 scalars
    print('  ' + ';  '.join(msg))


def _tensors(prefix, obj, out):
    if isinstance(obj, torch.Tensor):
        out[prefix] = obj.detach().clone()
    elif isinstance(obj, dict):
        for k, v in obj.items():
            _tensors(f'{prefix}.{k}', v, out)
    elif isinstance(obj, (tuple, list)):
        for k, v in enumerate(obj):
            _tensors(f'{prefix}.{k}', v, out)
    return out


def _snapshot(tr):
    """the packed weights of both engines (forward and backward packs, LoRA operands included) and the token table"""
    out = {}
    for tag, eng in (('unet', tr.engine), ('text', tr.text_engine)):
        _tensors(f'{tag}.w', eng.w, out)
        _tensors(f'{tag}.wb', getattr(eng, 'wb', {}), out)
    out['text.tok'] = tr.text_engine.tok.detach().clone()
    return out


@pytest.mark.parametrize('combo', COMBOS, ids=combo_id)
def test_train_loop_keeps_frozen_groups_bit_identical(cuda, tmp_path, monkeypatch, combo):
    import train_edlora as te
    emb_on, text_on, unet_on = combo
    from oracle import inject
    base, ref_unet, clip = _base_dir(tmp_path, clip_layers=1)
    tr = _trainer(base, combo)
    g = torch.Generator().manual_seed(1)
    m = torch.zeros(2, 1, 16, 16)
    m[:, :, 3:12, 4:13] = 1
    batch = {'images': torch.randn(2, 4, 16, 16, generator=g), 'prompts': ['photo of a <c1> <c2>', 'a <c1> <c2> smiling'],
             'masks': m, 'img_masks': torch.ones(2, 1, 16, 16)}
    tr._build(2)
    rows0 = tr._concept_rows().clone()
    w0 = _snapshot(tr)
    d0 = tr.delta_state_dict()
    logs = []
    counter = LaunchCounter(monkeypatch)
    # threshold above the rows' norm: the embedding learning rate decays without the freeze (tested elsewhere)
    te.train(tr, [batch] * 4, dataset_len=8, batch_size_per_gpu=2, print_freq=1, log=logs.append, emb_norm_threshold=10.0)
    monkeypatch.undo()
    # re-packs: one lora_pack per trained LoRA group per optimiser step, none for an absent one
    packs = collections.Counter(counter.lora_pack_tables)
    assert packs[tr.engine.lora_table.data_ptr()] == (4 if unet_on else 0)
    text_table = getattr(tr.text_engine, 'lora_table', None)
    assert (packs[text_table.data_ptr()] if text_table is not None else 0) == (4 if text_on else 0)
    assert sum(packs.values()) == 4 * (int(text_on) + int(unet_on))
    # the checkpoint: the reference's key sets for the trained LoRA groups (trainer_edlora.py:358-378), empty otherwise
    d1 = tr.delta_state_dict()
    assert set(d1) == {'new_concept_embedding', 'text_encoder', 'unet'} and list(d1['new_concept_embedding']) == ['<c1>', '<c2>']
    for part, on, model, where in (('text_encoder', text_on, clip, 'CLIPAttention'), ('unet', unet_on, ref_unet, 'Attention')):
        want = {f'{n}.lora_{s}.weight' for n in inject.lora_target_modules(model, where) for s in ('down', 'up')}
        assert set(d1[part]) == (want if on else set())
        if on:
            assert any(not torch.equal(d0[part][k], d1[part][k]) for k in d1[part])
    rows1 = tr._concept_rows()
    assert torch.equal(rows1, rows0) != emb_on
    w1 = _snapshot(tr)
    for k, v in w0.items():
        if k == 'text.tok':
            other = torch.ones(v.shape[0], dtype=torch.bool, device=v.device)
            other[49408:49408 + 32] = False
            assert torch.equal(w1[k][other], v[other]), 'non-concept rows moved'
            assert torch.equal(w1[k][~other], v[~other]) != emb_on
            continue
        is_lora = k.endswith('.lora_down') or k.endswith('.lora_up')
        owner = text_on if k.startswith('text.') else unet_on
        if not (is_lora and owner):
            assert torch.equal(w1[k], v), k              # base weights, and no LoRA operand of an absent group, move
    # the log: learning rates of the groups present (decayed linearly over 4 steps), then Norm_mean of the rows
    lrs = {'text_embedding': 1e-3, 'text_encoder': 1e-5, 'unet': 1e-4}
    for step, line in enumerate(logs):
        got = [float(x) for x in line.split(' lr ')[1].split(' Norm_mean ')[0].split(',')]
        assert got == pytest.approx([lrs[gname] * (4 - step) / 4 for gname in tr.groups], rel=1e-3)
    norms = [float(line.split('Norm_mean ')[1]) for line in logs]
    assert norms[-1] == pytest.approx(rows1.norm(dim=-1).mean().item(), rel=1e-3)
    if emb_on:
        assert norms[0] != norms[-1]
    else:                                                # constant rows: the same Norm_mean every step
        assert all(n == norms[0] for n in norms)
    # a checkpoint with a LoRA for a group this config does not train is refused, not silently dropped
    for part, on, model, where in (('text_encoder', text_on, clip, 'CLIPAttention'), ('unet', unet_on, ref_unet, 'Attention')):
        if not on:
            foreign = {'new_concept_embedding': {}, 'text_encoder': {}, 'unet': {},
                       part: inject.random_lora_state(model, seed=1, where=where)}
            with pytest.raises(ValueError, match='does not train'):
                tr.load_delta_state_dict(foreign)
    print(f'  {combo_id(combo)}: {logs[-1]}')


AUDITED = [(True, False, False), (False, True, False), (False, False, True), (True, False, True)]


@pytest.mark.parametrize('combo', AUDITED, ids=combo_id)
def test_new_launch_sequences_audited(cuda, tmp_path, combo):
    """one eager step and the optimiser step of each new engine configuration under the GEMM, attention and norm /
    elementwise launch audits: every launch against its float64 reference, its write window and a bit-identical rerun"""
    import attention_audit
    import gemm_audit
    import norm_audit
    from mos_b200 import dp
    base, ref_unet, clip = _base_dir(tmp_path, clip_layers=1)
    tr = _trainer(base, combo)
    tr._build(2)
    tr.engine.use_train_graph = False
    _, lat, noise, t, masks = _data(ref_unet, clip, combo)
    failures = []
    for mod in (gemm_audit, attention_audit, norm_audit):
        stats = gemm_audit.Stats()
        with mod.Recorder(stats):
            tr(lat, PROMPTS, masks, torch.ones_like(masks), noise=noise, timesteps=t)
            torch.cuda.synchronize()
        if mod is norm_audit:
            with mod.Recorder(stats):
                dp.optimizer_step(tr.state, 1.0, norm_out=torch.zeros(1, device='cuda'))
                torch.cuda.synchronize()
        assert stats.rows, mod.__name__
        print(f'\n{combo_id(combo)} {mod.__name__}\n' + stats.table())
        failures += stats.failures
    assert not failures, '\n'.join(failures[:30])


def test_train_opt_with_text_encoder_off(cuda, tmp_path, capsys):
    """`train_edlora.py -opt` on a shipped-style yml with text_encoder.enable_tuning: false: trains, writes
    edlora_model-latest.pth with an empty text_encoder section, validates from it, logs two learning rates and Norm_mean"""
    import train_edlora
    from synth import make_pretrained_dir
    from test_validation_sampling_gpu import _train_yml
    base = make_pretrained_dir(str(tmp_path / 'base'))
    yml = _train_yml(tmp_path, base, 'noclip', True)
    opt = yaml.safe_load(open(yml))
    opt['models']['finetune_cfg']['text_encoder']['enable_tuning'] = False
    open(yml, 'w').write(yaml.safe_dump(opt))
    losses = train_edlora.main(['-opt', yml])
    out = capsys.readouterr().out
    assert len(losses) == 4 and all(x == x for x in losses)
    ck = torch.load(tmp_path / 'noclip' / 'models' / 'edlora_model-latest.pth')['params']
    assert ck['text_encoder'] == {} and len(ck['unet']) > 0 and list(ck['new_concept_embedding']) == ['<c1>', '<c2>']
    lines = [l for l in out.splitlines() if l.startswith('iter ')]
    assert len(lines) == 4
    for k, line in enumerate(lines):
        lr = [float(x) for x in line.split(' lr ')[1].split(' Norm_mean ')[0].split(',')]
        assert lr == pytest.approx([1e-3 * (4 - k) / 4, 1e-4 * (4 - k) / 4], rel=1e-3)
        assert float(line.split('Norm_mean ')[1]) > 0
    assert 'load 0 LoRAs of text_encoder' in out
    root = tmp_path / 'noclip' / 'visualization' / 'PromptDataset'
    assert any(p.is_file() for p in root.rglob('*'))
    print('\n' + '\n'.join(lines))
