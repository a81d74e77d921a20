"""Host-side orchestration of gradient fusion (gradient_fusion.py:750-813 restated in mix-of-show_b200/gradient_fusion.py),
CPU only: checkpoint parsing, token / embedding bookkeeping, prompt construction and the inputs handed to the three
fusion stages.  The stages themselves (GPU) are replaced by recorders here; they have their own GPU parity tests."""
import json
import os

import torch

from oracle import inject
from oracle import unet as ou


class WordTokenizer:
    """whitespace tokenizer with CLIP's special ids and the calls the fusion code makes"""
    model_max_length = 77
    BOS, EOS = 49406, 49407

    def __init__(self):
        self.vocab = {}
        self.n = 49408

    def __len__(self):
        return self.n

    def add_tokens(self, names):
        added = 0
        for n in names:
            if n not in self.vocab:
                self.vocab[n] = self.n
                self.n += 1
                added += 1
        return added

    def convert_tokens_to_ids(self, name):
        return self.vocab.get(name, 0)         # unknown -> 0 (the unk id), as transformers tokenizers do

    def _ids(self, text):
        return [self.BOS] + [self.vocab.get(w, 1 + (sum(map(ord, w)) % 40000)) for w in text.split()] + [self.EOS]

    def save_pretrained(self, path):
        os.makedirs(path, exist_ok=True)
        json.dump({'added': sorted(self.vocab, key=self.vocab.get)}, open(os.path.join(path, 'word_tokenizer.json'), 'w'))

    @classmethod
    def from_pretrained(cls, path):
        t = cls()
        for w in json.load(open(os.path.join(path, 'word_tokenizer.json')))['added']:
            t.add_tokens([w])
        return t

    def __call__(self, text, padding='do_not_pad', max_length=77, truncation=True, return_tensors=None, **kw):
        from types import SimpleNamespace
        if isinstance(text, str):
            ids = self._ids(text)[:max_length]
            if padding == 'max_length':
                ids = ids + [self.EOS] * (max_length - len(ids))
            return SimpleNamespace(input_ids=torch.tensor([ids]) if return_tensors == 'pt' else ids)
        rows = [self._ids(t)[:max_length] for t in text]
        if padding == 'max_length':
            rows = [r + [self.EOS] * (max_length - len(r)) for r in rows]
        return SimpleNamespace(input_ids=torch.tensor(rows) if return_tensors == 'pt' else rows)


def test_compose_concepts_wiring(tmp_path, monkeypatch):
    import gradient_fusion as gf
    from transformers import CLIPTextConfig, CLIPTextModel
    from mixofshow.models.unet_b200 import UNet2DConditionModel
    from mixofshow.utils import model_io
    # ---- a tiny "pretrained" directory
    torch.manual_seed(0)
    unet = UNet2DConditionModel(block_out_channels=ou.TINY['block_out_channels'], layers_per_block=ou.TINY['layers_per_block'])
    base = str(tmp_path / 'base')
    model_io.save_unet(unet, base)
    clip = CLIPTextModel(CLIPTextConfig(vocab_size=49408, hidden_size=768, intermediate_size=3072, num_hidden_layers=1,
                                        num_attention_heads=12, max_position_embeddings=77)).eval()
    clip.save_pretrained(os.path.join(base, 'text_encoder'))
    # ---- two concept checkpoints in the reference's layout + the concept json
    ref_unet = ou.build_unet(0, ou.TINY)
    cfgs = []
    for c, name in enumerate(('<cat1> <cat2>', '<dog1>')):
        g = torch.Generator().manual_seed(c)
        params = {'new_concept_embedding': {w: torch.randn(16, 768, generator=g) for w in name.split()},
                  'text_encoder': inject.random_lora_state(clip, seed=c, where='CLIPAttention'),
                  'unet': inject.random_lora_state(ref_unet, seed=10 + c)}
        path = str(tmp_path / f'c{c}.pth')
        torch.save({'params': params}, path)
        cfgs.append({'lora_path': path, 'unet_alpha': 0.8 + 0.1 * c, 'text_encoder_alpha': 1.0, 'concept_name': name})
    cfg_path = str(tmp_path / 'concepts.json')
    json.dump(cfgs, open(cfg_path, 'w'))
    parsed = gf.parse_new_concepts(cfg_path)
    assert all(x is not None for part in parsed[:4] for x in part)
    assert all('attn2.to_k' in k or 'attn2.to_v' in k for k in parsed[2][0])
    assert not any('attn2.to_k' in k or 'attn2.to_v' in k for k in parsed[3][0])
    assert len(parsed[2][0]) + len(parsed[3][0]) == len(torch.load(cfgs[0]['lora_path'])['params']['unet'])
    # ---- stage recorders; the text encoder runs on CPU through transformers (same call shape as the GPU container)
    seen = {}
    monkeypatch.setattr(model_io, 'load_text_encoder',
                        lambda path, subfolder='text_encoder', **kw: CLIPTextModel.from_pretrained(os.path.join(path, subfolder)).eval())

    def fake_text(sd, lst, alphas, ids, iters, device='cuda', pad_id=49407):
        seen['text'] = (lst, alphas, ids, iters)
        k = 'text_model.encoder.layers.0.self_attn.q_proj.weight'
        return {k: sd[k] + 1.0}

    def fake_kv(sd, names, feats, lst, alphas, iters, device='cuda'):
        seen['kv'] = (names, feats, alphas, iters)
        return {names[0][1]: sd[names[0][1]] + 2.0}

    def fake_sp(sd, lst, alphas, embeds, iters, **kw):
        seen['sp'] = (alphas, embeds, iters, kw)
        k = 'mid_block.attentions.0.transformer_blocks.0.attn1.to_q.weight'
        return {k: sd[k] + 3.0}

    monkeypatch.setattr(gf, 'merge_text_encoder', fake_text)
    monkeypatch.setattr(gf, 'merge_kv_in_cross_attention', fake_kv)
    monkeypatch.setattr(gf, 'merge_spatial_attention', fake_sp)
    out_dir, new_cfg = gf.compose_concepts(cfg_path, 7, 3, base, str(tmp_path / 'out'), 'base', device='cpu',
                                           tokenizer=WordTokenizer(), log=lambda *a: None)
    # tokens: 16 per <word>, numbered consecutively over all concepts, ids after CLIP's vocabulary
    assert list(new_cfg) == ['<cat1>', '<cat2>', '<dog1>']
    assert new_cfg['<cat2>']['concept_token_names'] == [f'<new{16 + i}>' for i in range(16)]
    assert new_cfg['<dog1>']['concept_token_ids'] == list(range(49408 + 32, 49408 + 48))
    # text-encoder stage: per concept 32 un-padded sequences ('photo of a <c>' and '<c>' x 16 layers), alphas, iterations
    lst, alphas, ids, iters = seen['text']
    assert iters == 7 and alphas == [1.0, 1.0] and [len(x) for x in ids] == [32, 32]
    assert ids[0][0].tolist()[:1] == [49406] and ids[0][0].numel() == 7 and ids[0][16].numel() == 4   # BOS photo of a t t EOS
    assert ids[0][0][4].item() == 49408 and ids[0][1][4].item() == 49409                              # layer-bound tokens
    # cross-K/V stage: reference layer order, and per layer the features at the concept-token + EOS positions
    names, feats, alphas, iters = seen['kv']
    assert iters == 7 and alphas == [0.8, 0.9]
    assert [i for i, _ in names] == [0, 0, 1, 1, 2, 2, 3, 3] and names[0][1].endswith('attn2.to_k.weight') \
        and names[1][1].endswith('attn2.to_v.weight') and names[2][1].startswith('mid_block.')
    assert len(feats) == 2 and sorted(feats[0]) == list(range(16))
    assert feats[0][3].shape == (6, 768) and feats[1][3].shape == (4, 768)       # 2 prompts x (tokens + EOS)
    # spatial stage: one layer-wise embedding tensor per concept
    alphas, embeds, iters, kw = seen['sp']
    assert iters == 3 and embeds[0].shape == (1, 16, 77, 768) and kw['block_out'] == (320, 640)
    # ---- results folded back and written in the diffusers layout
    fused = model_io.load_unet(out_dir)
    k = 'mid_block.attentions.0.transformer_blocks.0.attn1.to_q.weight'
    assert torch.allclose(fused.state_dict()[k], unet.state_dict()[k] + 3.0)
    assert torch.allclose(fused.state_dict()[names[0][1]], unet.state_dict()[names[0][1]] + 2.0)
    te = CLIPTextModel.from_pretrained(os.path.join(out_dir, 'text_encoder'))
    assert te.get_input_embeddings().weight.shape[0] == 49408 + 48
    assert json.load(open(os.path.join(out_dir, 'new_concept_cfg.json'))) == new_cfg
    # ---- fuse -> reload -> tokenize round trip: the saved tokenizer knows the added tokens (a base tokenizer would split
    # '<new17>' into ordinary sub-tokens and the fused concept would silently be lost at sampling)
    tok = WordTokenizer.from_pretrained(os.path.join(out_dir, 'tokenizer'))
    model_io.ensure_concept_tokens(tok, new_cfg)
    from mixofshow.pipelines.pipeline_edlora import bind_concept_prompt
    p0 = bind_concept_prompt('photo of a <cat1> <cat2>', new_cfg)
    ids0 = tok(p0[3], padding='max_length', max_length=77, return_tensors='pt').input_ids[0].tolist()
    assert new_cfg['<cat1>']['concept_token_ids'][3] in ids0 and new_cfg['<cat2>']['concept_token_ids'][3] in ids0
    base_tok = WordTokenizer()                                   # the BASE tokenizer: tokens are re-added in id order
    model_io.ensure_concept_tokens(base_tok, new_cfg)
    assert base_tok.convert_tokens_to_ids('<new47>') == 49408 + 47
    shifted = WordTokenizer()
    shifted.add_tokens(['<other>'])                              # ids no longer line up -> loud failure
    import pytest
    with pytest.raises(ValueError):
        model_io.ensure_concept_tokens(shifted, new_cfg)
