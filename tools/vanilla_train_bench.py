"""Time one full-size SD1.5 training step at batch 4 (config 2: 512 x 512 images, 64 x 64 latents, synthetic weights,
all three parameter groups: concept rows, rank-4 CLIPAttention LoRA, rank-4 Attention LoRA, the attention regulariser),
ED-LoRA next to vanilla LoRA (`enable_edlora: false`: B text sequences instead of 16 B, one embedding shared by the 16
cross-attention layers, d(text embedding) summed over them in fp32).

One step = the captured forward + loss + backward (text encoder and UNet) replayed from its CUDA graph, then the flat AdamW
step and the LoRA re-packs (tools/finetune_groups_bench.py's step), timed with CUDA events after a warm-up.  The two
modes are measured alternately, `--rounds` times each, and one JSON line is printed per measurement with the card name
and power limit read in the same process.

    python tools/vanilla_train_bench.py [--steps 20] [--warmup 5] [--rounds 2]
"""
import argparse
import json
import math
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, 'mix-of-show_b200'), os.path.join(ROOT, 'tests'), os.path.join(ROOT, 'tools')):
    if p not in sys.path:
        sys.path.insert(0, p)

import torch  # noqa: E402

B = 4


def build(vanilla):
    """the engines EDLoRATrainer._build makes for all three groups, ED-LoRA (32 concept rows, 16 B text sequences) or
    vanilla LoRA (2 concept rows, B text sequences)"""
    from types import SimpleNamespace

    import bench
    from mos_b200 import dp
    from mos_b200.clip_train_engine import CLIPTrainEngine
    from mos_b200.train_engine import TrainEngine
    sd, lora, _, _, _ = bench.build_workload()
    dev = torch.device('cuda')
    tsd = bench.synthetic_clip_state()
    g0 = torch.Generator().manual_seed(12)
    tlora = {}
    for i in range(12):
        for pj in ('q_proj', 'k_proj', 'v_proj', 'out_proj'):
            m = f'text_model.encoder.layers.{i}.self_attn.{pj}'
            tlora[m + '.lora_down.weight'] = (torch.rand(4, 768, generator=g0) * 2 - 1) / math.sqrt(768)
            tlora[m + '.lora_up.weight'] = torch.randn(768, 4, generator=g0) * 0.02
    ids = list(range(49408, 49408 + (2 if vanilla else 32)))
    n_unet = sum(v.numel() for v in lora.values())
    state = dp.FlatTrainState(len(ids), 768, CLIPTrainEngine.lora_param_count(12, 768, 960), n_unet,
                              lrs=(1e-3, 1e-5, 1e-4), device=dev)
    eng = TrainEngine(sd, B, 64, 64, lora=lora, attn_reg_weight=0.01, reg_full_identity=False, state=state,
                      state_offset=state.group_end[1], text_grad=True, device=dev, shared_ehs=vanilla)
    nx = len(eng.xattn_names)
    te = CLIPTrainEngine(tsd, (1 if vanilla else nx) * B, lora=tlora, concept_token_ids=ids, state=state, emb_offset=0,
                         lora_offset=state.group_end[0], device=dev)
    eng.attach_text_engine(te)
    return SimpleNamespace(eng=eng, text=te, state=state, B=B, nx=nx, concept_ids=ids, text_grad=True, vanilla=vanilla)


def inputs(w, seed):
    """tests/engine_walks.train_sd15_full_inputs; vanilla: the ids of layer 0 with the two concept tokens <new0> <new1>"""
    from engine_walks import train_sd15_full_inputs
    if not w.vanilla:
        return train_sd15_full_inputs(w, seed)
    ed = train_sd15_full_inputs(type(w)(B=w.B, nx=1, concept_ids=list(range(49408, 49408 + 32))), seed)
    ids = ed['text_ids'].clone()
    ids[:, 2], ids[:, 3] = w.concept_ids
    return dict(ed, text_ids=ids)


def main(argv=None):
    from finetune_groups_bench import card, step
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=20)
    ap.add_argument('--warmup', type=int, default=5)
    ap.add_argument('--rounds', type=int, default=2)
    a = ap.parse_args(argv)
    assert torch.cuda.is_available(), 'timing needs the GPU'
    name, power = card()
    for r in range(a.rounds):
        for vanilla in (False, True):
            w = build(vanilla)
            batches = [inputs(w, 100 + i) for i in range(4)]
            norm = torch.zeros(1, device='cuda')
            for i in range(a.warmup):
                step(w, batches[i % 4], norm)
            torch.cuda.synchronize()
            times = []
            for i in range(a.steps):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                step(w, batches[i % 4], norm)
                e1.record()
                e1.synchronize()
                times.append(e0.elapsed_time(e1))
            times.sort()
            print(json.dumps({'mode': 'vanilla' if vanilla else 'edlora', 'round': r, 'batch': B,
                              'text_sequences': w.text.n_seq, 'median_ms': round(times[len(times) // 2], 3),
                              'min_ms': round(times[0], 3), 'steps': a.steps, 'warmup': a.warmup, 'gpu': name,
                              'power_limit': power}), flush=True)
            del w, batches
            torch.cuda.empty_cache()


if __name__ == '__main__':
    main()
