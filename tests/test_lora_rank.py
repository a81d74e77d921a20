"""LoRA ranks 1-3 on the host side of training (CPU only): the rank bounds of `lora_cfg.rank`, the flat training state
(four rank slots per module whatever the rank, so its size does not depend on the rank), and the refusal of a LoRA
whose rank is not the configured rank of its group.

The flat state would load such a LoRA without complaint: a rank-4 checkpoint under `rank: 2` fills all four slots,
trains four ranks and saves two; a rank-2 checkpoint under `rank: 4` trains two ranks and saves two zero rows.  The
reference raises there (it copies each tensor into a parameter of the configured shape), and so must this trainer,
before any engine is built."""
import copy

import pytest
import torch

from oracle import inject
from test_finetune_groups import base, finetune_cfg  # noqa: F401  (module fixture)

PLACEMENTS = [('CLIPAttention', 'Attention'), ('CLIPEncoderLayer', 'Transformer2DModel')]
PLACEMENT_IDS = ['attention', 'whole_block']


def _cfg(text_rank, unet_rank, wheres=PLACEMENTS[0]):
    cfg = finetune_cfg(True, True, True, *wheres)
    cfg['text_encoder']['lora_cfg']['rank'] = text_rank
    cfg['unet']['lora_cfg']['rank'] = unet_rank
    return cfg


def _trainer(path, cfg):
    from test_fusion_orchestration import WordTokenizer
    from mixofshow.pipelines.trainer_edlora import EDLoRATrainer
    return EDLoRATrainer(path, '<c1>+<c2>', '<rand-0.02>+<rand-0.02>', True, finetune_cfg=copy.deepcopy(cfg),
                         tokenizer=WordTokenizer(), device='cpu')


def _delta(ref_unet, clip, text_rank, unet_rank, wheres=PLACEMENTS[0]):
    return {'new_concept_embedding': {},
            'text_encoder': inject.random_lora_state(clip, seed=3, rank=text_rank, where=wheres[0]),
            'unet': inject.random_lora_state(ref_unet, seed=4, rank=unet_rank, where=wheres[1])}


@pytest.mark.parametrize('wheres', PLACEMENTS, ids=PLACEMENT_IDS)
@pytest.mark.parametrize('part', ['text_encoder', 'unet'])
@pytest.mark.parametrize('ckpt_rank,cfg_rank', [(4, 2), (2, 4), (1, 3), (3, 1)])
def test_checkpoint_of_another_rank_refused(base, wheres, part, ckpt_rank, cfg_rank):
    """a whole group at the wrong rank, with the other group at its configured rank"""
    path, ref_unet, clip = base
    ranks = {'text_encoder': 2, 'unet': 2, part: cfg_rank}
    tr = _trainer(path, _cfg(ranks['text_encoder'], ranks['unet'], wheres))
    delta = _delta(ref_unet, clip, ranks['text_encoder'], ranks['unet'], wheres)
    tr.load_delta_state_dict(copy.deepcopy(delta))                  # the configured ranks load (deferred to the build)
    assert tr._loaded is not None
    tr._loaded = None
    model = clip if part == 'text_encoder' else ref_unet
    delta[part] = inject.random_lora_state(model, seed=5, rank=ckpt_rank, where=wheres[part == 'unet'])
    first = next(iter(delta[part]))[:-len('.lora_down.weight')]
    with pytest.raises(ValueError, match=rf'{part} LoRA of {first}: .*rank {ckpt_rank}, the config trains rank {cfg_rank}'):
        tr.load_delta_state_dict(delta)
    assert tr._loaded is None and tr.engine is None


@pytest.mark.parametrize('wheres', PLACEMENTS, ids=PLACEMENT_IDS)
@pytest.mark.parametrize('part', ['text_encoder', 'unet'])
@pytest.mark.parametrize('ckpt_rank,cfg_rank', [(4, 2), (2, 4)])
def test_one_module_of_another_rank_refused(base, wheres, part, ckpt_rank, cfg_rank):
    """every tensor is checked, not a sample: the LAST module of the reference's walk at the wrong rank (proj_out's 4-D
    [r, K, 1, 1] / [N, r, 1, 1] pair with `where: Transformer2DModel`, mlp.fc2 with CLIPEncoderLayer)"""
    path, ref_unet, clip = base
    tr = _trainer(path, _cfg(cfg_rank, cfg_rank, wheres))
    delta = _delta(ref_unet, clip, cfg_rank, cfg_rank, wheres)
    model = clip if part == 'text_encoder' else ref_unet
    other = inject.random_lora_state(model, seed=6, rank=ckpt_rank, where=wheres[part == 'unet'])
    last = list(delta[part])[-1][:-len('.lora_up.weight')]
    assert last.endswith({'Transformer2DModel': 'proj_out', 'CLIPEncoderLayer': 'mlp.fc2'}.get(wheres[part == 'unet'],
                                                                                             last.split('.')[-1]))
    for s in ('down', 'up'):
        delta[part][f'{last}.lora_{s}.weight'] = other[f'{last}.lora_{s}.weight']
    if last.endswith('proj_out'):
        assert delta[part][f'{last}.lora_down.weight'].shape == (ckpt_rank, 320, 1, 1)
        want = rf'lora_down \({ckpt_rank}, 320, 1, 1\), lora_up \(320, {ckpt_rank}, 1, 1\)'
    else:
        want = rf'lora_down \({ckpt_rank}, \d+\), lora_up \(\d+, {ckpt_rank}\)'
    with pytest.raises(ValueError, match=rf'{part} LoRA of {last}: {want}: rank {ckpt_rank}, the config trains rank {cfg_rank}'):
        tr.load_delta_state_dict(delta)
    assert tr._loaded is None


@pytest.mark.parametrize('part', ['text_encoder', 'unet'])
@pytest.mark.parametrize('down_rank,up_rank', [(2, 4), (4, 2), (1, 3)])
def test_down_and_up_of_different_ranks_refused(base, part, down_rank, up_rank):
    path, ref_unet, clip = base
    for cfg_rank in (down_rank, up_rank):
        tr = _trainer(path, _cfg(cfg_rank, cfg_rank))
        delta = _delta(ref_unet, clip, cfg_rank, cfg_rank)
        m = list(delta[part])[2][:-len('.lora_down.weight')]
        K, N = delta[part][m + '.lora_down.weight'].shape[1], delta[part][m + '.lora_up.weight'].shape[0]
        delta[part][m + '.lora_down.weight'] = torch.randn(down_rank, K)
        delta[part][m + '.lora_up.weight'] = torch.randn(N, up_rank)
        with pytest.raises(ValueError, match=rf'{part} LoRA of {m}: lora_down \({down_rank}, \d+\), lora_up \(\d+, {up_rank}\): '
                                             rf'down and up disagree on the rank, the config trains rank {cfg_rank}'):
            tr.load_delta_state_dict(delta)


@pytest.mark.parametrize('rank', [1, 2, 3, 4])
def test_matching_ranks_accepted_by_check(base, rank):
    from mixofshow.pipelines.trainer_edlora import check_lora_ranks
    _, ref_unet, clip = base
    for part, model, where in (('unet', ref_unet, 'Transformer2DModel'), ('text_encoder', clip, 'CLIPEncoderLayer')):
        lora = inject.random_lora_state(model, rank=rank, where=where)
        check_lora_ranks(lora, rank, part)
        with pytest.raises(ValueError, match=f'rank {rank}, the config trains rank {rank % 4 + 1}'):
            check_lora_ranks(lora, rank % 4 + 1, part)
    check_lora_ranks({}, rank, 'unet')                     # an empty section has nothing to refuse


def test_rank_of_untrained_group_not_checked(base):
    """a LoRA for a group the config does not train is refused for that reason when it is applied, whatever its rank"""
    path, ref_unet, clip = base
    cfg = finetune_cfg(True, False, True)
    cfg['unet']['lora_cfg']['rank'] = 2
    tr = _trainer(path, cfg)
    delta = _delta(ref_unet, clip, 3, 2)
    tr.load_delta_state_dict(delta)                       # deferred: the rank of the untrained group is not checked
    assert tr._loaded is delta


def test_unet_lora_trainer_refuses_lora_state_of_another_rank():
    """UNetLoRATrainer checks the `lora_state` it hands to its TrainEngine before the engine is built"""
    from mixofshow.pipelines.trainer_edlora import UNetLoRATrainer
    from oracle import unet as ou
    ref = ou.build_unet(0, ou.TINY)
    cfg = {'unet': {'enable_tuning': True, 'lr': 1e-4, 'lora_cfg': {'rank': 2, 'alpha': 1.0, 'where': 'Attention'}}}
    topo = dict(block_out=ou.TINY['block_out_channels'], layers=ou.TINY['layers_per_block'])
    with pytest.raises(ValueError, match=r'unet LoRA of down_blocks\.0\..*: rank 4, the config trains rank 2'):
        UNetLoRATrainer(ref.state_dict(), 2, finetune_cfg=cfg, unet_topology=topo, device='cpu',
                        lora_state=inject.random_lora_state(ref, rank=4))


@pytest.mark.parametrize('rank', [0, 5, -1, 16])
def test_rank_bounds_refused(base, rank):
    from mixofshow.pipelines.trainer_edlora import _check_rank
    path, _, _ = base
    with pytest.raises(ValueError, match='rank must be in 1..4'):
        _check_rank({'rank': rank})
    for text_rank, unet_rank in ((rank, 4), (4, rank)):
        with pytest.raises(ValueError, match='rank must be in 1..4'):
            _trainer(path, _cfg(text_rank, unet_rank))


@pytest.mark.parametrize('wheres', PLACEMENTS, ids=PLACEMENT_IDS)
def test_ranks_accepted_and_flat_sizes_rank_independent(base, wheres):
    from mixofshow.pipelines.trainer_edlora import _check_rank
    path, _, _ = base
    sizes = {}
    for rank in (1, 2, 3, 4):
        assert _check_rank({'rank': rank, 'alpha': 0.5}) == (rank, 0.5)
        tr = _trainer(path, _cfg(rank, 5 - rank if rank > 1 else 1, wheres))
        assert (tr.text_rank, tr.unet_rank) == (rank, 5 - rank if rank > 1 else 1)
        sizes[rank] = tr.flat_group_sizes()
    assert len(set(sizes.values())) == 1, sizes
    assert all(n > 0 for n in sizes[1])


@pytest.mark.parametrize('rank', [1, 2, 4])
def test_convert_merge_of_1x1_convs_at_rank(rank):
    """convert_edlora's merge of a whole-block LoRA (the weights test_edlora.py and validation sample with) against float64
    W + alpha up @ down, proj_in / proj_out included: at rank 1 squeezing the [N, 1, 1, 1] / [1, K, 1, 1] pair would
    turn up @ down into a dot product added to every element"""
    from mixofshow.utils.convert_edlora_to_diffusers import merge_lora_into_weight
    from oracle import unet as ou
    sd = ou.build_unet(0, ou.TINY).state_dict()
    lora = inject.random_lora_state(ou.build_unet(0, ou.TINY), seed=2, rank=rank, where='Transformer2DModel', up_std=0.05)
    out = merge_lora_into_weight(sd, lora, 'unet', 0.7)
    names = [k[:-len('.lora_down.weight')] for k in lora if k.endswith('.lora_down.weight')]
    assert any(n.endswith('proj_in') for n in names)
    for m in names:
        W = sd[m + '.weight']
        up, down = lora[m + '.lora_up.weight'].double(), lora[m + '.lora_down.weight'].double()
        want = W.double() + 0.7 * (up.flatten(1) @ down.flatten(1)).view(W.shape)
        assert out[m + '.weight'].shape == W.shape
        assert (out[m + '.weight'].double() - want).abs().max().item() < 1e-6, m
