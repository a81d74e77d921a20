"""Time the full-size SD1.5 ED-LoRA training step at batch 2 for four parameter-group configurations (trainer_edlora.py
:70-142): all three groups, UNet LoRA only, embedding rows only, text-encoder LoRA only.

One step = the captured forward + loss + backward (text encoder and UNet) replayed from its CUDA graph, then the flat AdamW
step and the LoRA re-packs, timed with CUDA events after a warm-up; prints one JSON line per configuration with the card
name and power limit read in the same process.

    python tools/finetune_groups_bench.py [--steps 20] [--warmup 5] [--configs all,unet,emb,text]
"""
import argparse
import json
import math
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, 'mix-of-show_b200'), os.path.join(ROOT, 'tests')):
    if p not in sys.path:
        sys.path.insert(0, p)

import torch  # noqa: E402

CONFIGS = {'all': (True, True, True), 'unet': (False, False, True), 'emb': (True, False, False),
           'text': (False, True, False)}


def build(combo, B=2):
    """the engines EDLoRATrainer._build makes for `combo` = (embedding rows, text LoRA, UNet LoRA) on bench.py's SD1.5
    workload (rank-4 `where: Attention` / `CLIPAttention` LoRAs, the regulariser on all 16 cross layers)"""
    from types import SimpleNamespace

    import bench
    from mos_b200 import dp
    from mos_b200.clip_engine import CLIPTextEngine
    from mos_b200.clip_train_engine import CLIPTrainEngine
    from mos_b200.train_engine import TrainEngine
    emb, text, unet = combo
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
    ids = list(range(49408, 49408 + 32))
    n_text = CLIPTrainEngine.lora_param_count(12, 768, 960) if text else 0
    n_unet = sum(v.numel() for v in lora.values()) if unet else 0
    state = dp.FlatTrainState(len(ids) if emb else 0, 768, n_text, n_unet, lrs=(1e-3, 1e-5, 1e-4), device=dev)
    text_grad = emb or text
    eng = TrainEngine(sd, B, 64, 64, lora=lora if unet else None, attn_reg_weight=0.01, reg_full_identity=False,
                      state=state, state_offset=state.group_end[1], text_grad=text_grad, device=dev)
    nx = len(eng.xattn_names)
    if text_grad:
        te = CLIPTrainEngine(tsd, nx * B, lora=tlora if text else None, concept_token_ids=ids, state=state,
                             emb_offset=0 if emb else None, lora_offset=state.group_end[0], device=dev)
    else:
        te = CLIPTextEngine(tsd, nx * B, device=dev)
    if not emb:
        state.set_const_rows(te.tok[torch.tensor(ids, device=dev)])
    eng.attach_text_engine(te)
    return SimpleNamespace(eng=eng, text=te, state=state, B=B, nx=nx, concept_ids=ids, text_grad=text_grad)


def step(w, batch, norm):
    from mos_b200 import dp
    w.eng.forward_backward(**batch)
    scale = dp.allreduce_flat_device(w.state, w.eng.loss_out[0:1])
    dp.optimizer_step(w.state, scale, norm_out=norm)
    w.eng.refresh_lora()
    if w.text_grad:
        w.text.refresh_lora()


def card():
    name = torch.cuda.get_device_name(0)
    try:
        out = subprocess.run(['nvidia-smi', '--query-gpu=power.limit', '--format=csv,noheader', '-i', '0'],
                             capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        out = 'unknown'
    return name, out


def main(argv=None):
    from engine_walks import train_sd15_full_inputs
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=20)
    ap.add_argument('--warmup', type=int, default=5)
    ap.add_argument('--configs', default='all,unet,emb,text')
    a = ap.parse_args(argv)
    assert torch.cuda.is_available(), 'timing needs the GPU'
    name, power = card()
    for cfg in a.configs.split(','):
        w = build(CONFIGS[cfg])
        batches = [train_sd15_full_inputs(w, 100 + i) for i in range(4)]
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
        print(json.dumps({'config': cfg, 'groups': CONFIGS[cfg], 'batch': w.B, 'median_ms': round(times[len(times) // 2], 3),
                          'min_ms': round(times[0], 3), 'steps': a.steps, 'warmup': a.warmup, 'gpu': name,
                          'power_limit': power}), flush=True)
        del w, batches
        torch.cuda.empty_cache()


if __name__ == '__main__':
    main()
