"""Host side of the LoRA placements (`lora_cfg.where`, trainer_edlora.py:100-133), on the CPU: which modules carry a LoRA
for each placement (against oracle.inject.lora_target_modules, the reference's module walk), the flat-state and checkpoint
parameter counts at SD1.5 sizes, the GEGLU row-order round trip, and the values the trainers accept."""
import json

import pytest
import torch


def _sd15_unet_meta():
    from oracle import unet as ou
    with torch.device('meta'):
        return ou.UNet2DConditionModel(None)


def _count(state):
    return sum(v.numel() for v in state.values())


@pytest.mark.parametrize('where', ['Attention', 'Transformer2DModel'])
@pytest.mark.parametrize('topo', ['tiny', 'sd15'])
def test_unet_module_names_match_reference_walk(where, topo):
    from mixofshow.pipelines.trainer_edlora import _NameProbe
    from mos_b200.train_engine import TrainEngine
    from oracle import inject
    from oracle import unet as ou
    if topo == 'tiny':
        ref = ou.build_unet(0, ou.TINY)
        t = dict(block_out=ou.TINY['block_out_channels'], layers=ou.TINY['layers_per_block'])
    else:
        ref, t = _sd15_unet_meta(), {}
    names = TrainEngine.lora_module_names.__get__(_NameProbe(t, where))()
    assert names == inject.lora_target_modules(ref, where)


def test_unet_parameter_counts_sd15():
    from oracle import inject
    ref = _sd15_unet_meta()
    mods = dict(ref.named_modules())

    def count(where):
        n = 0
        for m in inject.lora_target_modules(ref, where):
            w = mods[m].weight
            n += 4 * (w[0].numel() + w.shape[0])
        return n
    assert count('Attention') == 797184
    assert count('Transformer2DModel') == 1695744              # 797 184 + 898 560


def test_clip_module_names_and_counts():
    from transformers import CLIPTextConfig, CLIPTextModel
    from mos_b200.clip_train_engine import CLIPTrainEngine
    from oracle import inject
    for where in ('CLIPAttention', 'CLIPEncoderLayer'):
        m = CLIPTextModel(CLIPTextConfig(vocab_size=1000, hidden_size=768, intermediate_size=3072, num_hidden_layers=2,
                                         num_attention_heads=12, max_position_embeddings=77))
        want = inject.random_lora_state(m, where=where)
        names = CLIPTrainEngine.module_names(2, where)
        assert sorted(f'{n}.lora_{p}.weight' for n in names for p in ('down', 'up')) == sorted(want)
    # 12 layers at SD1.5 sizes, rank 4: checkpoint and flat (pads included) parameter counts
    per_layer_attn = 4 * (4 * 768 + 4 * 768)
    per_layer_mlp = 4 * (768 + 3072) + 4 * (3072 + 768)
    assert 12 * per_layer_attn == 294912 and 12 * per_layer_mlp == 368640
    assert 12 * (per_layer_attn + per_layer_mlp) == 663552
    assert CLIPTrainEngine.lora_param_count(12, 768, 960) == 331776
    assert CLIPTrainEngine.lora_param_count(12, 768, 960, where='CLIPEncoderLayer') == 331776 + 12 * (
        4 * (768 + 3200) + 4 * (3200 + 768))


def test_geglu_perm_round_trip():
    from mos_b200.engine import geglu_perm
    for n in (2560, 5120, 10240):
        perm = geglu_perm(n)
        assert sorted(perm.tolist()) == list(range(n))
        u = torch.randn(n, 4)
        packed = u[perm]
        back = torch.empty_like(packed)
        back[perm] = packed
        assert torch.equal(back, u)
        # tile t holds value rows 80t..80t+79, then the gate rows H + 80t ..
        assert perm[80:160].tolist() == list(range(n // 2, n // 2 + 80))


def test_trainers_accept_exactly_the_reference_placements():
    from mixofshow.pipelines.trainer_edlora import EDLoRATrainer, UNetLoRATrainer
    base = {'text_embedding': {'enable_tuning': True, 'lr': 1e-3},
            'text_encoder': {'enable_tuning': True, 'lora_cfg': {'rank': 4, 'alpha': 1.0}, 'lr': 1e-5},
            'unet': {'enable_tuning': True, 'lora_cfg': {'rank': 4, 'alpha': 1.0}, 'lr': 1e-4}}
    for tw in ('CLIPAttention', 'CLIPEncoderLayer', 'Attention', 'Linear'):
        for uw in ('Attention', 'Transformer2DModel', 'CLIPAttention', 'BasicTransformerBlock'):
            cfg = json.loads(json.dumps(base))
            cfg['text_encoder']['lora_cfg']['where'] = tw
            cfg['unet']['lora_cfg']['where'] = uw
            tr = object.__new__(EDLoRATrainer)
            if tw in ('CLIPAttention', 'CLIPEncoderLayer') and uw in ('Attention', 'Transformer2DModel'):
                tr.set_finetune_cfg(cfg)
                assert (tr.text_where, tr.unet_where) == (tw, uw)
            else:
                with pytest.raises(NotImplementedError):
                    tr.set_finetune_cfg(cfg)
    ucfg = {'unet': {'enable_tuning': True, 'lr': 1e-4, 'lora_cfg': {'rank': 4, 'alpha': 1.0, 'where': 'CLIPAttention'}}}
    with pytest.raises(NotImplementedError):
        UNetLoRATrainer({}, 1, finetune_cfg=ucfg)
