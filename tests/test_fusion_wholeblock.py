"""Host side of gradient fusion for the whole-block LoRA placements (`where: Transformer2DModel` / `CLIPEncoderLayer`): the
weight name -> engine record key mapping both fusion stages use, the checkpoint check that runs before any stage, and the
split of a checkpoint into its cross-K/V and spatial parts."""
import pytest
import torch
from transformers import CLIPTextConfig, CLIPTextModel

import gradient_fusion as gf
from oracle import inject
from oracle import unet as ou

TN = 'down_blocks.1.attentions.0'
TB = TN + '.transformer_blocks.0'
LAYER = 'text_model.encoder.layers.3'

# every leaf kind a fusion stage solves -> the input the engine records for it
RECORD = {
    f'{TB}.attn1.to_q.weight': f'{TB}.attn1.in',
    f'{TB}.attn1.to_k.weight': f'{TB}.attn1.in',
    f'{TB}.attn1.to_v.weight': f'{TB}.attn1.in',
    f'{TB}.attn1.to_out.0.weight': f'{TB}.attn1.to_out.0',
    f'{TB}.attn2.to_q.weight': f'{TB}.attn2.to_q',
    f'{TB}.attn2.to_out.0.weight': f'{TB}.attn2.to_out.0',
    f'{TB}.ff.net.0.proj.weight': f'{TB}.ff.net.0.proj',
    f'{TB}.ff.net.2.weight': f'{TB}.ff.net.2',
    f'{TN}.proj_in.weight': f'{TN}.proj_in',
    f'{TN}.proj_out.weight': f'{TN}.proj_out',
    f'{LAYER}.self_attn.q_proj.weight': f'{LAYER}.self_attn.in',
    f'{LAYER}.self_attn.k_proj.weight': f'{LAYER}.self_attn.in',
    f'{LAYER}.self_attn.v_proj.weight': f'{LAYER}.self_attn.in',
    f'{LAYER}.self_attn.out_proj.weight': f'{LAYER}.self_attn.out_proj',
    f'{LAYER}.mlp.fc1.weight': f'{LAYER}.mlp.fc1',
    f'{LAYER}.mlp.fc2.weight': f'{LAYER}.mlp.fc2',
}


def _clip(layers=1):
    torch.manual_seed(0)
    return CLIPTextModel(CLIPTextConfig(vocab_size=1000, hidden_size=768, intermediate_size=3072,
                                        num_hidden_layers=layers, num_attention_heads=12, max_position_embeddings=77)).eval()


@pytest.mark.parametrize('name', sorted(RECORD))
def test_record_key_of_every_leaf_kind(name):
    assert gf.record_key(name) == RECORD[name]
    assert gf.record_key(name[:-len('.weight')]) == RECORD[name]      # module names map the same way


@pytest.mark.parametrize('name', [f'{TB}.attn2.to_k.weight', f'{TB}.attn2.to_v.weight',
                                  'down_blocks.0.resnets.0.conv1.weight', f'{TB}.norm1.weight'])
def test_record_key_refuses_layers_without_a_recorded_input(name):
    with pytest.raises(KeyError, match='no recorded input'):
        gf.record_key(name)


def test_record_keys_cover_whole_block_checkpoints():
    """every spatial / text weight of a whole-block checkpoint has a record key, with the 10 UNet and 6 CLIP kinds"""
    unet, clip = ou.build_unet(0, ou.TINY), _clip()
    u = inject.random_lora_state(unet, where='Transformer2DModel')
    t = inject.random_lora_state(clip, where='CLIPEncoderLayer')
    spatial = {k.replace('.lora_down', '') for k in u if k.endswith('lora_down.weight') and 'attn2.to_k' not in k
               and 'attn2.to_v' not in k}
    text = {k.replace('.lora_down', '') for k in t if k.endswith('lora_down.weight')}
    assert len(spatial) == 4 * 10 and len(text) == 6
    keys = {gf.record_key(n) for n in spatial}
    assert len(keys) == 4 * 8                        # q|k|v of attn1 share one input
    assert len({gf.record_key(n) for n in text}) == 4


def test_check_lora_targets_accepts_whole_block_and_refuses_other_layers():
    unet, clip = ou.build_unet(0, ou.TINY), _clip()
    for uw, tw in (('Attention', 'CLIPAttention'), ('Transformer2DModel', 'CLIPEncoderLayer'),
                   ('Transformer2DModel', 'CLIPAttention'), ('Attention', 'CLIPEncoderLayer')):
        gf._check_lora_targets({'unet': inject.random_lora_state(unet, where=uw),
                                'text_encoder': inject.random_lora_state(clip, where=tw)}, 'ok.pth')
    params = {'unet': inject.random_lora_state(unet, where='Transformer2DModel'), 'text_encoder': {}}
    params['unet']['down_blocks.0.resnets.0.conv1.lora_down.weight'] = torch.zeros(4, 320, 3, 3)
    params['unet']['down_blocks.0.resnets.0.conv1.lora_up.weight'] = torch.zeros(320, 4, 1, 1)
    with pytest.raises(ValueError, match=r'bad\.pth.*resnets\.0\.conv1\.lora_'):
        gf._check_lora_targets(params, 'bad.pth')
    te = inject.random_lora_state(clip, where='CLIPEncoderLayer')
    te['text_model.encoder.layers.0.layer_norm1.lora_down.weight'] = torch.zeros(4, 768)
    with pytest.raises(ValueError, match='layer_norm1'):
        gf._check_lora_targets({'text_encoder': te}, 'bad.pth')


def test_parse_new_concepts_splits_whole_block_checkpoints(tmp_path):
    unet, clip = ou.build_unet(0, ou.TINY), _clip()
    params = {'new_concept_embedding': {'<c1>': torch.zeros(16, 768)},
              'unet': inject.random_lora_state(unet, where='Transformer2DModel'),
              'text_encoder': inject.random_lora_state(clip, where='CLIPEncoderLayer')}
    path = str(tmp_path / 'c.pth')
    torch.save({'params': params}, path)
    emb, te, kv, sp, _ = gf.parse_new_concepts([{'lora_path': path, 'concept_name': '<c1>'}])
    kv, sp = kv[0], sp[0]
    assert set(kv) | set(sp) == set(params['unet']) and not set(kv) & set(sp)
    assert kv and all(('attn2.to_k.' in k or 'attn2.to_v.' in k) for k in kv)
    assert len(kv) == 4 * 2 * 2                      # 4 cross-attentions x (to_k, to_v) x (down, up)
    for kind in ('ff.net.0.proj', 'ff.net.2', 'proj_in', 'proj_out'):
        assert sum(f'.{kind}.lora_' in k for k in sp) == 4 * 2, kind
    assert sp['down_blocks.0.attentions.0.proj_in.lora_down.weight'].ndim == 4
    assert set(te[0]) == set(params['text_encoder'])
    assert list(emb[0]) == ['<c1>']
