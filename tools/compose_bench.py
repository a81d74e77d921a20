"""BASELINE config 3 END TO END on one H100: `gradient_fusion.compose_concepts` (the entry point `python gradient_fusion.py`
drives) on a synthetic SD1.5-size model directory and 5 synthetic ED-LoRA concept checkpoints in the reference's
on-disk layout - load, token / embedding merge, text-encoder merge (48 CLIPAttention linears x 500 L-BFGS iterations),
cross-attention K/V merge (32 x 500), spatial-attention merge (96 x 50, incl. the recorded UNet forwards), save and
re-load of the fused model.  Prints one JSON line with the wall-clock seconds of every stage.

    python tools/compose_bench.py [--concepts 5] [--textenc-iters 500] [--unet-iters 50] [--tiny]
"""
import argparse
import json
import os
import shutil
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, 'mix-of-show_b200')]
import torch  # noqa: E402

import bench  # noqa: E402


class WordTokenizer:
    """Whitespace tokenizer with CLIP's special ids and the calls the fusion code makes (there are no CLIP vocabulary files
    in this image; the fusion only needs ids, `add_tokens`, `save_pretrained`)."""
    model_max_length = 77
    BOS, EOS = 49406, 49407

    def __init__(self):
        self.vocab, self.n = {}, 49408

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
        return self.vocab.get(name, 0)

    def _ids(self, text):
        return [self.BOS] + [self.vocab.get(w, 1 + (sum(map(ord, w)) % 40000)) for w in text.split()] + [self.EOS]

    def save_pretrained(self, path):
        os.makedirs(path, exist_ok=True)
        json.dump({'added': sorted(self.vocab, key=self.vocab.get)}, open(os.path.join(path, 'word_tokenizer.json'), 'w'))

    def __call__(self, text, padding='do_not_pad', max_length=77, truncation=True, return_tensors=None, **kw):
        from types import SimpleNamespace
        single = isinstance(text, str)
        rows = [self._ids(t)[:max_length] for t in ([text] if single else text)]
        if padding == 'max_length':
            rows = [r + [self.EOS] * (max_length - len(r)) for r in rows]
        if return_tensors == 'pt':
            return SimpleNamespace(input_ids=torch.tensor(rows))
        return SimpleNamespace(input_ids=rows[0] if single else rows)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--concepts', type=int, default=5)
    ap.add_argument('--textenc-iters', type=int, default=500)       # fuse.sh / gradient_fusion.py defaults
    ap.add_argument('--unet-iters', type=int, default=50)
    ap.add_argument('--tiny', action='store_true')
    a = ap.parse_args()
    import gradient_fusion as gf
    from mixofshow.models.unet_b200 import UNet2DConditionModel
    from mixofshow.utils import model_io
    from transformers import CLIPTextConfig, CLIPTextModel
    work = tempfile.mkdtemp(prefix='compose_bench_')
    out = {'config': f'gradient_fusion.compose_concepts, {a.concepts} synthetic ED-LoRAs, '
                     f'{"tiny" if a.tiny else "SD1.5-size"} UNet + 12-layer CLIP text encoder, 1xH100',
           'textenc_iters': a.textenc_iters, 'unet_iters': a.unet_iters}
    try:
        t0 = time.perf_counter()
        sd, _, _, _, cfg = bench.build_workload(a.tiny)
        unet = UNet2DConditionModel(**(cfg or {}))
        unet.load_state_dict(sd)
        base = os.path.join(work, 'base')
        model_io.save_unet(unet, base)
        torch.manual_seed(1)
        clip = CLIPTextModel(CLIPTextConfig(vocab_size=49408, hidden_size=768, intermediate_size=3072, num_hidden_layers=12,
                                            num_attention_heads=12, max_position_embeddings=77, hidden_act='quick_gelu')).eval()
        clip.save_pretrained(os.path.join(base, 'text_encoder'))
        cfgs = []
        for c in range(a.concepts):
            g = torch.Generator().manual_seed(50 + c)
            words = [f'<c{c}a>', f'<c{c}b>']
            tlora = {}
            for i in range(12):
                for pj in ('q_proj', 'k_proj', 'v_proj', 'out_proj'):
                    m = f'text_model.encoder.layers.{i}.self_attn.{pj}'
                    tlora[m + '.lora_down.weight'] = (torch.rand(4, 768, generator=g) * 2 - 1) / 768 ** 0.5
                    tlora[m + '.lora_up.weight'] = torch.randn(768, 4, generator=g) * 0.02
            params = {'new_concept_embedding': {w: torch.randn(16, 768, generator=g) * 0.02 for w in words},
                      'text_encoder': tlora, 'unet': bench.random_unet_lora(sd, cfg, seed=10 + c)}
            path = os.path.join(work, f'concept{c}.pth')
            torch.save({'params': params}, path)
            cfgs.append({'lora_path': path, 'unet_alpha': 1.0, 'text_encoder_alpha': 1.0, 'concept_name': ' '.join(words)})
        cfg_path = os.path.join(work, 'concepts.json')
        json.dump(cfgs, open(cfg_path, 'w'))
        del unet, clip
        out['setup_seconds'] = round(time.perf_counter() - t0, 2)
        stamps = []

        def log(msg, *rest):
            torch.cuda.synchronize()
            stamps.append((time.perf_counter(), str(msg)))

        t1 = time.perf_counter()
        out_dir, new_cfg = gf.compose_concepts(cfg_path, a.textenc_iters, a.unet_iters, base, os.path.join(work, 'out'), 'bench',
                                               device='cuda', tokenizer=WordTokenizer(), log=log)
        torch.cuda.synchronize()
        t2 = time.perf_counter()
        stamps.append((t2, 'end'))
        stage = {}
        for (ta, name), (tb, _) in zip(stamps[:-1], stamps[1:]):
            key = name.strip('-')
            stage[key] = round(tb - ta, 2)
        out['stage_seconds'] = stage
        out['compose_concepts_seconds'] = round(t2 - t1, 2)
        out['new_concept_tokens'] = sum(len(v['concept_token_ids']) for v in new_cfg.values())
        # the fused directory must load again (from_pretrained layout) and carry finite weights
        fused = model_io.load_unet(out_dir)
        w = fused.state_dict()['down_blocks.0.attentions.0.transformer_blocks.0.attn2.to_k.weight']
        out['fused_reload_ok'] = bool(torch.isfinite(w).all())
        d0 = sd['down_blocks.0.attentions.0.transformer_blocks.0.attn2.to_k.weight']
        out['example_crosskv_delta_rel'] = round(((w.float().cpu() - d0).norm() / d0.norm()).item(), 5)
        out['data'] = 'synthetic (random-init weights, random LoRAs up ~ N(0, 0.02^2), whitespace tokenizer stub)'
    finally:
        shutil.rmtree(work, ignore_errors=True)
    print(json.dumps(out))


if __name__ == '__main__':
    main()
