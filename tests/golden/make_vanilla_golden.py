"""Generate tests/golden/vanilla_golden.pt by executing the REFERENCE's own Python (read-only, in place, under the import
shims of oracle/ref_shims.py) for vanilla LoRA (`enable_edlora: false`).  Run where the reference exists:
    python tests/golden/make_vanilla_golden.py
Pinned here:
  - `EDLoRATrainer.cal_attn_reg` (trainer_edlora.py:263-313) with ONE id row per sample (l = 1: the prompts are not
    bound, :220-221): loss, autograd gradients of the two concept columns, the concept-token positions;
  - `load_new_concept(pipe, emb, enable_edlora=False)` (convert_edlora_to_diffusers.py:4-31): one token `<new{idx}>` per
    concept, its id and the row written into the embedding table.
The fixture is data only; tests/test_vanilla_lora.py checks the oracle (oracle/train_ref.py) and the product against it.
"""
import math
import os
import sys
import types

import torch
import torch.nn as nn

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(HERE))
from oracle import ref_shims  # noqa: E402
from oracle.train_ref import attn_reg_inputs  # noqa: E402

OUT = os.path.join(HERE, 'vanilla_golden.pt')
CONCEPT_IDS = (49408, 49409)            # <new0>, <new1>: one token per concept


def vanilla_attn_reg_inputs():
    """the maps and masks of oracle.train_ref.attn_reg_inputs with unbound ids [b, 77]: <new0> and <new1> once each"""
    maps, masks, _, pos = attn_reg_inputs()
    ids = torch.full((2, 77), 49407, dtype=torch.long)
    ids[:, 0] = 49406
    for i, (p0, p1) in enumerate(pos):
        ids[i, p0], ids[i, p1] = CONCEPT_IDS
    return maps, masks, ids, pos


def golden_attn_reg():
    tr = ref_shims.load_reference_module('mixofshow/pipelines/trainer_edlora.py')
    out = {}
    for full in (True, False):
        maps, masks, ids, pos = vanilla_attn_reg_inputs()
        for lst in maps.values():
            for m in lst:
                m.requires_grad_(True)
        me = types.SimpleNamespace(get_all_concept_token_ids=lambda: list(CONCEPT_IDS), reg_full_identity=full,
                                   attn_reg_weight=0.01)
        loss = tr.EDLoRATrainer.cal_attn_reg(me, maps, masks, ids)
        loss.backward()
        grads = {}
        for lst in maps.values():
            for m in lst:
                r = int(math.sqrt(m.shape[1]))
                g = m.grad.view(2, 8, r * r, 77)
                grads[r] = torch.stack([g[i][0][:, pos[i]] for i in range(2)]).clone()      # [b, N, 2]
        out['full' if full else 'masked'] = dict(loss=loss.detach(), grads=grads)
    out['pos'] = pos
    return out


def golden_load_new_concept():
    from test_fusion_orchestration import WordTokenizer
    conv = ref_shims.load_reference_module('mixofshow/utils/convert_edlora_to_diffusers.py')

    class TextEncoder:
        def __init__(self):
            self.emb = nn.Embedding(49408, 768)
            nn.init.zeros_(self.emb.weight)

        def resize_token_embeddings(self, n):
            old = self.emb.weight.data
            self.emb = nn.Embedding(n, old.shape[1])
            self.emb.weight.data.zero_()
            self.emb.weight.data[:old.shape[0]] = old

        def get_input_embeddings(self):
            return self.emb

    g = torch.Generator().manual_seed(11)
    emb = {'<cat1>': torch.randn(1, 768, generator=g) * 0.02, '<dog2>': torch.randn(1, 768, generator=g) * 0.02}
    pipe = types.SimpleNamespace(tokenizer=WordTokenizer(), text_encoder=TextEncoder())
    pipe, cfg = conv.load_new_concept(pipe, emb, enable_edlora=False)
    table = pipe.text_encoder.get_input_embeddings().weight.data
    return dict(embedding=emb, new_concept_cfg=cfg, n_vocab=len(pipe.tokenizer), rows=table[49408:].clone())


def main():
    if not ref_shims.reference_available():
        raise SystemExit(f'the reference is not at {ref_shims.REFERENCE_ROOT}')
    torch.save({'attn_reg_l1': golden_attn_reg(), 'load_new_concept': golden_load_new_concept()}, OUT)
    print('wrote', OUT)


if __name__ == '__main__':
    main()
