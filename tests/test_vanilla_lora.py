"""Vanilla LoRA (`models.enable_edlora: false`) on the host side: the reference's import line, one token `<new{k}>` per
concept, unbound [b, 77] tokenization and the concept positions of the attention regulariser, the flat-state size, the
`lora_model-*.pth` checkpoint names, the refusals (validation during training, test_edlora.py, gradient fusion), the
StableDiffusionPipeline prompt encoding, and the oracle / product against the reference's own `cal_attn_reg` (l = 1) and
`load_new_concept(enable_edlora=False)` pinned by tests/golden/vanilla_golden.pt (tests/golden/make_vanilla_golden.py)."""
import math
import os
import types

import pytest
import torch
import yaml

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'vanilla_golden.pt')
FINETUNE = {'text_embedding': {'enable_tuning': True, 'lr': 1e-3},
            'text_encoder': {'enable_tuning': False},
            'unet': {'enable_tuning': True, 'lora_cfg': {'rank': 4, 'alpha': 1.0, 'where': 'Attention'}, 'lr': 1e-4}}


@pytest.fixture(scope='module')
def base(tmp_path_factory):
    from synth import make_pretrained_dir
    return make_pretrained_dir(str(tmp_path_factory.mktemp('vanilla') / 'base'), clip_layers=1, with_vae=False)


def _trainer(base, enable_edlora, init='<rand-0.02>+a'):
    from mixofshow.pipelines.trainer_edlora import EDLoRATrainer
    return EDLoRATrainer(base, '<c1>+<c2>', init, enable_edlora, finetune_cfg=FINETUNE, device='cpu',
                         latent_size=(16, 16), attn_reg_weight=0.01)


@pytest.fixture(scope='module')
def golden():
    return torch.load(GOLDEN)


def test_reference_import_line_resolves():
    # test_edlora.py:16 / train_edlora.py:18 of the reference
    from mixofshow.pipelines.pipeline_edlora import EDLoRAPipeline, StableDiffusionPipeline
    assert callable(StableDiffusionPipeline.from_pretrained) and callable(EDLoRAPipeline.from_pretrained)
    assert not hasattr(StableDiffusionPipeline, 'set_new_concept_cfg')          # as in diffusers
    assert hasattr(EDLoRAPipeline, 'set_new_concept_cfg')


def test_one_token_per_concept(base):
    tr = _trainer(base, False)
    assert tr.enable_edlora is False
    assert tr.new_concept_cfg == {'<c1>': {'concept_token_ids': [49408], 'concept_token_names': ['<new0>']},
                                  '<c2>': {'concept_token_ids': [49409], 'concept_token_names': ['<new1>']}}
    tok = tr.text_encoder.get_input_embeddings().weight.data
    a_id = tr.tokenizer.encode('a', add_special_tokens=False)[0]
    assert torch.equal(tok[49409], tok[a_id])                                     # initialised from an existing token
    assert 0 < tok[49408].norm() < 2 * 0.02 * math.sqrt(768)                      # <rand-0.02>
    ed = _trainer(base, True)
    assert [c['concept_token_names'][-1] for c in ed.new_concept_cfg.values()] == ['<new15>', '<new31>']


def test_flat_state_has_one_row_per_concept(base):
    van, ed = _trainer(base, False), _trainer(base, True)
    assert van.flat_group_sizes()[0] == 2 * 768
    assert ed.flat_group_sizes()[0] == 32 * 768
    assert van.flat_group_sizes()[1:] == ed.flat_group_sizes()[1:]


def test_tokenization_is_unbound(base):
    from oracle import train_ref
    tr = _trainer(base, False)
    prompts = ['photo of a <new0> <new1>', 'a <new0> <new1> on a beach']
    ids = tr.tokenize(prompts)
    assert ids.shape == (2, 77)
    assert torch.equal(ids, tr.tokenizer(prompts, padding='max_length', max_length=77, truncation=True,
                                         return_tensors='pt').input_ids)
    pos = tr.concept_token_positions(ids, 2)
    assert pos == train_ref.concept_token_positions(ids, 2, tr.get_all_concept_token_ids())
    for row, (p0, p1) in zip(ids, pos):
        assert (int(row[p0]), int(row[p1])) == (49408, 49409)
    # the shipped `<TOK>: <potter1> <potter2>` style mapping names the concepts, not their tokens: no concept position
    with pytest.raises(ValueError, match='exactly two concept tokens'):
        tr.concept_token_positions(tr.tokenize(['photo of a <c1> <c2>', 'a <c1> <c2>']), 2)


def _opt(tmp_path, enable_edlora, val_during_save):
    return {'name': 'v', 'models': {'pretrained_path': str(tmp_path / 'missing'), 'enable_edlora': enable_edlora},
            'datasets': {'train': {'path': str(tmp_path / 'missing.pt'), 'batch_size_per_gpu': 1}},
            'train': {'optim_g': {'type': 'AdamW', 'lr': 0.0}},
            'val': {'val_during_save': val_during_save},
            'path': {'models': str(tmp_path / 'models')}}


def test_train_refuses_validating_vanilla_lora_at_startup(tmp_path):
    import train_edlora
    yml = tmp_path / 'lora.yml'
    yml.write_text(yaml.safe_dump(_opt(tmp_path, False, True)))
    # refused before CUDA, the model directory or the data set are touched (none of them exists here)
    with pytest.raises(NotImplementedError, match='val_during_save.*enable_edlora=False'):
        train_edlora.main(['-opt', str(yml)])
    train_edlora.check_options(_opt(tmp_path, False, False))
    train_edlora.check_options(_opt(tmp_path, True, True))


def test_checkpoint_names(tmp_path):
    import train_edlora
    opt = _opt(tmp_path, False, False)
    assert train_edlora.checkpoint_path(opt, 3) == str(tmp_path / 'models' / 'lora_model-3.pth')
    assert train_edlora.checkpoint_path(opt, 'latest') == str(tmp_path / 'models' / 'lora_model-latest.pth')
    assert train_edlora.checkpoint_path(_opt(tmp_path, True, False), 3).endswith('edlora_model-3.pth')
    delta = {'new_concept_embedding': {'<c1>': torch.zeros(1, 768)}, 'text_encoder': {}, 'unet': {}}
    trainer = types.SimpleNamespace(delta_state_dict=lambda: delta)
    train_edlora.save_and_validation(trainer, opt, None, 'latest', log=lambda *a: None)
    assert os.listdir(tmp_path / 'models') == ['lora_model-latest.pth']
    assert torch.load(tmp_path / 'models' / 'lora_model-latest.pth')['params']['new_concept_embedding']['<c1>'].shape == (1, 768)


def test_test_edlora_points_to_stable_diffusion_pipeline():
    import test_edlora
    with pytest.raises(NotImplementedError, match='enable_edlora=False') as e:
        test_edlora.check_edlora({'models': {'enable_edlora': False}})
    assert 'StableDiffusionPipeline' in str(e.value) and 'convert_edlora' in str(e.value)


def test_fusion_refuses_vanilla_checkpoint(tmp_path):
    import gradient_fusion as gf
    path = str(tmp_path / 'lora_model-latest.pth')
    torch.save({'params': {'new_concept_embedding': {'<c1>': torch.zeros(1, 768)}, 'text_encoder': {}, 'unet': {}}}, path)
    with pytest.raises(ValueError, match=f'{path}.*1 rows'):
        gf.parse_new_concepts([{'lora_path': path, 'concept_name': '<c1>'}])


def test_stable_diffusion_pipeline_encodes_prompts_unbound():
    from test_fusion_orchestration import WordTokenizer
    from mixofshow.pipelines.pipeline_edlora import StableDiffusionPipeline
    calls = []

    def text_encoder(ids):
        calls.append(ids.clone())
        return (ids[:, :, None].float().expand(-1, -1, 768) / 1e5,)

    tok = WordTokenizer()
    tok.add_tokens(['<new0>'])
    pipe = StableDiffusionPipeline(text_encoder=text_encoder, tokenizer=tok, unet=object()).to('cpu')
    emb = pipe._encode_prompt(['a <new0> dog', 'a cat'], 'cpu', 1, True, negative_prompt=['ugly', 'blurry'])
    assert emb.shape == (4, 77, 768)
    assert [c.shape for c in calls] == [(2, 77), (2, 77)]                          # one CLIP pass per prompt, no binding
    assert int(calls[0][0, 2]) == 49408 and int(calls[0][0, 3]) != 49408
    assert torch.equal(emb[2:], text_encoder(calls[0])[0]) and torch.equal(emb[:2], text_encoder(calls[1])[0])
    assert pipe._encode_prompt(None, 'cpu', 1, False, prompt_embeds=emb[2:]).shape == (2, 77, 768)
    with pytest.raises(ValueError, match=r'\[B, 77, 768\]'):
        pipe._encode_prompt(None, 'cpu', 1, False, prompt_embeds=emb[2:, None])


def test_oracle_attn_reg_l1_vs_reference_golden(golden):
    """oracle.train_ref.concept_token_positions / cal_attn_reg on unbound ids [b, 77] vs the reference's cal_attn_reg"""
    from oracle import train_ref as tr
    g = golden['attn_reg_l1']
    maps, masks, _, pos = tr.attn_reg_inputs()
    ids = torch.full((2, 77), 49407, dtype=torch.long)
    ids[:, 0] = 49406
    for i, (p0, p1) in enumerate(pos):
        ids[i, p0], ids[i, p1] = 49408, 49409
    got_pos = tr.concept_token_positions(ids, 2, [49408, 49409])
    assert got_pos == g['pos'] == pos
    for tag, full in (('full', True), ('masked', False)):
        maps, masks, _, _ = tr.attn_reg_inputs()
        for lst in maps.values():
            for m in lst:
                m.requires_grad_(True)
        loss = tr.cal_attn_reg(maps, masks, got_pos, reg_full_identity=full, attn_reg_weight=0.01)
        assert abs(loss.item() - g[tag]['loss'].item()) <= 1e-6 * abs(g[tag]['loss'].item())
        loss.backward()
        for lst in maps.values():
            for m in lst:
                r = int(math.sqrt(m.shape[1]))
                gr = m.grad.view(2, 8, r * r, 77)
                gc = torch.stack([gr[i][0][:, pos[i]] for i in range(2)])
                ref = g[tag]['grads'][r].float()
                assert (gc - ref).abs().max().item() <= 1e-6 * ref.abs().max().item()


def test_load_new_concept_vanilla_vs_reference_golden(golden):
    from test_fusion_orchestration import WordTokenizer
    from mixofshow.utils.convert_edlora_to_diffusers import load_new_concept
    g = golden['load_new_concept']

    class TextEncoder:
        def __init__(self):
            self.emb = torch.nn.Embedding(49408, 768)
            torch.nn.init.zeros_(self.emb.weight)

        def resize_token_embeddings(self, n):
            old = self.emb.weight.data
            self.emb = torch.nn.Embedding(n, old.shape[1])
            self.emb.weight.data.zero_()
            self.emb.weight.data[:old.shape[0]] = old

        def get_input_embeddings(self):
            return self.emb

    pipe = types.SimpleNamespace(tokenizer=WordTokenizer(), text_encoder=TextEncoder())
    pipe, cfg = load_new_concept(pipe, g['embedding'], enable_edlora=False)
    assert cfg == g['new_concept_cfg'] and len(pipe.tokenizer) == g['n_vocab']
    assert torch.equal(pipe.text_encoder.get_input_embeddings().weight.data[49408:], g['rows'])
