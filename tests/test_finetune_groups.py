"""EDLoRATrainer.set_finetune_cfg for every non-empty subset of ED-LoRA's three parameter groups (trainer_edlora.py:70-142),
CPU only: the optimizer's parameter groups and learning rates, the sizes of the flat training state, the checkpoint's
LoRA key sets, the all-off rejection, and convert_edlora on a checkpoint whose LoRA sections are empty."""
import copy
import itertools
import os

import pytest
import torch

from oracle import inject
from oracle import unet as ou

LRS = {'text_embedding': 1e-3, 'text_encoder': 1e-5, 'unet': 1e-4}
GROUPS = ('text_embedding', 'text_encoder', 'unet')
COMBOS = [c for c in itertools.product((False, True), repeat=3) if any(c)]


def finetune_cfg(emb, text, unet, text_where='CLIPAttention', unet_where='Attention'):
    """a shipped-style finetune_cfg with each group's enable_tuning flag set as given (the LoRA groups keep their lora_cfg)"""
    return {'text_embedding': {'enable_tuning': emb, 'lr': LRS['text_embedding']},
            'text_encoder': {'enable_tuning': text, 'lr': LRS['text_encoder'],
                             'lora_cfg': {'rank': 4, 'alpha': 1.0, 'where': text_where}},
            'unet': {'enable_tuning': unet, 'lr': LRS['unet'], 'lora_cfg': {'rank': 4, 'alpha': 1.0, 'where': unet_where}}}


def combo_id(c):
    return '+'.join(g for g, on in zip(GROUPS, c) if on)


@pytest.fixture(scope='module')
def base(tmp_path_factory):
    """tiny 2-level UNet (the oracle's TINY topology) and a 1-layer CLIP text encoder at SD1.5 widths"""
    from transformers import CLIPTextConfig, CLIPTextModel
    from mixofshow.models.unet_b200 import UNet2DConditionModel
    from mixofshow.utils import model_io
    torch.manual_seed(0)
    ref_unet = ou.build_unet(0, ou.TINY)
    unet = UNet2DConditionModel(block_out_channels=ou.TINY['block_out_channels'], layers_per_block=ou.TINY['layers_per_block'])
    unet.load_state_dict(ref_unet.state_dict())
    path = str(tmp_path_factory.mktemp('finetune_groups') / 'base')
    model_io.save_unet(unet, path)
    clip = CLIPTextModel(CLIPTextConfig(vocab_size=49408, hidden_size=768, intermediate_size=3072, num_hidden_layers=1,
                                        num_attention_heads=12, max_position_embeddings=77)).eval()
    clip.save_pretrained(os.path.join(path, 'text_encoder'))
    return path, ref_unet, clip


def _trainer(path, cfg):
    from test_fusion_orchestration import WordTokenizer
    from mixofshow.pipelines.trainer_edlora import EDLoRATrainer
    return EDLoRATrainer(path, '<c1>+<c2>', '<rand-0.02>+<rand-0.02>', True, finetune_cfg=copy.deepcopy(cfg),
                         tokenizer=WordTokenizer(), device='cpu')


def _reference_keys(model, where):
    """checkpoint keys of the reference's LoRA walk (trainer_edlora.py:100-133, 371-378)"""
    return {f'{n}.lora_{s}.weight' for n in inject.lora_target_modules(model, where) for s in ('down', 'up')}


@pytest.mark.parametrize('combo', COMBOS, ids=combo_id)
@pytest.mark.parametrize('wheres', [('CLIPAttention', 'Attention'), ('CLIPEncoderLayer', 'Transformer2DModel')],
                         ids=['attention', 'whole_block'])
def test_groups_sizes_and_checkpoint_keys(base, combo, wheres):
    path, ref_unet, clip = base
    emb, text, unet = combo
    cfg = finetune_cfg(emb, text, unet, *wheres)
    tr = _trainer(path, cfg)
    # parameter groups: the enabled ones, in the order embedding -> text LoRA -> UNet LoRA, with their learning rates
    assert tr.groups == tuple(g for g, on in zip(GROUPS, combo) if on)
    assert [g['lr'] for g in tr.get_params_to_optimize()] == [LRS[g] for g in tr.groups]
    # flat state [concept rows | text LoRA | UNet LoRA]: an absent group has zero length
    names = tr.lora_module_names()
    n_rows, n_text, n_unet = tr.flat_group_sizes()
    assert n_rows == (32 * 768 if emb else 0)
    ca = 12 * 80                                 # CLIP heads run padded to 80 dims; mlp.fc1 rows 3072 -> 3200
    per_layer = 3 * 4 * (768 + ca) + 4 * (ca + 768) + (4 * (768 + 3200) * 2 if wheres[0] == 'CLIPEncoderLayer' else 0)
    assert n_text == (per_layer if text else 0)
    usd = ref_unet.state_dict()
    want_unet = sum(4 * (usd[m + '.weight'][0].numel() + usd[m + '.weight'].shape[0])
                    for m in inject.lora_target_modules(ref_unet, wheres[1]))
    assert n_unet == (want_unet if unet else 0)
    # checkpoint LoRA sections: the reference's module walk for a trained group, empty otherwise
    keys = {part: {f'{m}.lora_{s}.weight' for m in names[part] for s in ('down', 'up')} for part in names}
    assert keys['text_encoder'] == (_reference_keys(clip, wheres[0]) if text else set())
    assert keys['unet'] == (_reference_keys(ref_unet, wheres[1]) if unet else set())
    # the 16 tokens per concept are added whatever the flags say (init_new_concept, :55)
    assert tr.get_all_concept_token_ids() == list(range(49408, 49408 + 32))


def test_all_groups_off_rejected(base):
    path, _, _ = base
    with pytest.raises(ValueError, match='no parameter group'):
        _trainer(path, finetune_cfg(False, False, False))
    # a LoRA group without a lora_cfg does not train (trainer_edlora.py:97, 118)
    cfg = finetune_cfg(False, True, True)
    del cfg['text_encoder']['lora_cfg'], cfg['unet']['lora_cfg']
    with pytest.raises(ValueError, match='no parameter group'):
        _trainer(path, cfg)


def test_where_and_rank_checked_only_for_trained_groups(base):
    path, _, _ = base
    cfg = finetune_cfg(True, False, True)
    cfg['text_encoder']['lora_cfg'] = {'rank': 9, 'where': 'Nowhere'}
    assert _trainer(path, cfg).groups == ('text_embedding', 'unet')
    cfg['unet']['lora_cfg']['rank'] = 9
    with pytest.raises(ValueError, match='rank'):
        _trainer(path, cfg)
    cfg = finetune_cfg(False, True, False, text_where='Nowhere')
    with pytest.raises(NotImplementedError, match='where'):
        _trainer(path, cfg)


def _convert(convert_edlora, ckpt, clip, ref_unet):
    from types import SimpleNamespace
    from test_checkpoint_formats import FakeTokenizer
    from transformers import CLIPTextConfig, CLIPTextModel
    torch.manual_seed(0)
    te = CLIPTextModel(CLIPTextConfig(vocab_size=300, hidden_size=768, intermediate_size=3072, num_hidden_layers=1,
                                      num_attention_heads=12, max_position_embeddings=77))
    te.load_state_dict(clip)
    un = ou.build_unet(0, ou.TINY)
    un.load_state_dict(ref_unet)
    pipe = SimpleNamespace(tokenizer=FakeTokenizer(300), text_encoder=te, unet=un)
    pipe, cfg = convert_edlora(pipe, copy.deepcopy(ckpt), enable_edlora=True, alpha=0.7)
    return cfg, te.state_dict(), un.state_dict()


@pytest.mark.parametrize('empty', [('text_encoder',), ('unet',), ('text_encoder', 'unet')], ids='+'.join)
def test_convert_edlora_with_empty_lora_sections(empty, capsys):
    """A checkpoint of a run with a LoRA group off merges 0 LoRAs of that network: its weights are the pretrained ones,
    bit for bit, and the concept rows are still loaded (convert_edlora_to_diffusers.py:79-99)."""
    from test_checkpoint_formats import _clip_sd, _delta
    from mixofshow.utils.convert_edlora_to_diffusers import convert_edlora
    ref_unet = ou.build_unet(0, ou.TINY)
    clip, clip_sd = _clip_sd()
    ckpt = _delta(ref_unet, clip, seed=3)
    for part in empty:
        ckpt['params'][part] = {}
    unet_sd = {k: v.clone() for k, v in ref_unet.state_dict().items()}
    cfg, te, un = _convert(convert_edlora, ckpt, clip_sd, unet_sd)
    out = capsys.readouterr().out
    for part, got, base in (('text_encoder', te, clip_sd), ('unet', un, unet_sd)):
        changed = [k for k in base if not torch.equal(got[k], base[k])]
        if part in empty:
            assert f'load 0 LoRAs of {part}' in out
            assert changed == [] or changed == ['text_model.embeddings.token_embedding.weight']
        else:
            assert len(changed) >= len(ckpt['params'][part]) // 2
    assert list(cfg) == ['<cat1>', '<dog2>']
    rows = te['text_model.embeddings.token_embedding.weight'][300:]
    assert torch.equal(rows, torch.cat([ckpt['params']['new_concept_embedding'][c] for c in cfg]))
    from oracle import ref_shims
    if not ref_shims.reference_available():
        return
    ref = ref_shims.load_reference_module('mixofshow/utils/convert_edlora_to_diffusers.py')
    cfg_r, te_r, un_r = _convert(ref.convert_edlora, ckpt, clip_sd, unet_sd)
    assert cfg_r == cfg
    for a, b in ((te, te_r), (un, un_r)):
        assert sorted(a) == sorted(b) and all(torch.equal(a[k], b[k]) for k in a)
