"""BASELINE config 3 END TO END on one H100: `gradient_fusion.compose_concepts` (the entry point `python gradient_fusion.py`
drives) on a synthetic SD1.5-size model directory and 5 synthetic ED-LoRA concept checkpoints in the reference's
on-disk layout - load, token / embedding merge, text-encoder merge (48 CLIPAttention linears x 500 L-BFGS iterations;
72 with `--text-where CLIPEncoderLayer`), cross-attention K/V merge (32 x 500), spatial merge (96 x 50, incl. the recorded
UNet forwards; 160 with `--unet-where Transformer2DModel`), save and re-load of the fused model.  Prints one JSON line with
the wall-clock seconds of every stage and the card they were measured on.

    python tools/compose_bench.py [--concepts 5] [--textenc-iters 500] [--unet-iters 50] [--tiny]
                                  [--unet-where {Attention,Transformer2DModel}] [--text-where {CLIPAttention,CLIPEncoderLayer}]

Under `torchrun --nproc-per-node N` the layer solves are sharded over the ranks (gradient_fusion.fusion_plan); the stage
seconds are then the maximum over the ranks, and `plan` gives every rank's layer count and share of the planned cost per
stage.
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


def _lora_pair(g, W, rank=4):
    """random rank-4 pair for the weight W ([out, in], or a 1x1 conv [out, in, 1, 1]) in the trainer's checkpoint shapes:
    down ~ kaiming-uniform(a=sqrt(5)), up ~ N(0, 0.02^2) (as bench.random_unet_lora)"""
    cout, cin, tail = W.shape[0], W.shape[1], tuple(W.shape[2:])
    down = ((torch.rand(rank, cin, generator=g) * 2 - 1) / cin ** 0.5).reshape(rank, cin, *tail)
    up = (torch.randn(cout, rank, generator=g) * 0.02).reshape(cout, rank, *tail)
    return down, up


def whole_block_unet_lora(sd, cfg, seed):
    """`where: Transformer2DModel`: the attention LoRA of bench.random_unet_lora plus proj_in / proj_out (1x1 convs, saved
    4-D) and ff.net.0.proj / ff.net.2 of every transformer block"""
    from mos_b200.engine import cross_attention_names
    lora = bench.random_unet_lora(sd, cfg, seed=seed)
    g = torch.Generator().manual_seed(1000 + seed)
    names = cross_attention_names(cfg['block_out_channels'], cfg['layers_per_block']) if cfg else cross_attention_names()
    for an in names:
        tn = an[:-len('.transformer_blocks.0.attn2')]
        for m in (f'{tn}.proj_in', f'{tn}.transformer_blocks.0.ff.net.0.proj', f'{tn}.transformer_blocks.0.ff.net.2',
                  f'{tn}.proj_out'):
            lora[m + '.lora_down.weight'], lora[m + '.lora_up.weight'] = _lora_pair(g, sd[m + '.weight'])
    return lora


def gpu_card():
    """name and power limit of the GPU the stages run on (the power limit bounds the clocks under sustained load)"""
    import subprocess
    name = torch.cuda.get_device_name()
    try:
        limit = subprocess.run(['nvidia-smi', '--query-gpu=power.limit', '--format=csv,noheader', '-i',
                                str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        limit = ''
    return {'name': name, 'power_limit': limit or 'unknown'}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--concepts', type=int, default=5)
    ap.add_argument('--textenc-iters', type=int, default=500)       # fuse.sh / gradient_fusion.py defaults
    ap.add_argument('--unet-iters', type=int, default=50)
    ap.add_argument('--tiny', action='store_true')
    ap.add_argument('--unet-where', choices=('Attention', 'Transformer2DModel'), default='Attention')
    ap.add_argument('--text-where', choices=('CLIPAttention', 'CLIPEncoderLayer'), default='CLIPAttention')
    a = ap.parse_args()
    import torch.distributed as dist
    import gradient_fusion as gf
    from mos_b200 import dp
    rank, world, device = gf.init_distributed()
    plans = []
    fusion_plan = gf.fusion_plan

    def plan_and_note(shapes, iters, w):
        plans.append((shapes, iters, fusion_plan(shapes, iters, w)))
        return plans[-1][2]

    gf.fusion_plan = plan_and_note
    work = [tempfile.mkdtemp(prefix='compose_bench_') if rank == 0 else None]
    if world > 1:
        dist.broadcast_object_list(work)
    work = work[0]
    out = {'config': f'gradient_fusion.compose_concepts, {a.concepts} synthetic ED-LoRAs, '
                     f'{"tiny" if a.tiny else "SD1.5-size"} UNet + 12-layer CLIP text encoder, {world} rank(s) on '
                     f'{torch.cuda.device_count()} visible H100(s)',
           'world_size': world, 'textenc_iters': a.textenc_iters, 'unet_iters': a.unet_iters, 'unet_where': a.unet_where,
           'text_where': a.text_where, 'gpu': gpu_card()}
    try:
        if rank == 0:
            write_workload(a, work, out)
        if world > 1:
            dist.barrier()
        stamps = []

        def log(msg, *rest):
            torch.cuda.synchronize()
            stamps.append((time.perf_counter(), str(msg)))

        t1 = time.perf_counter()
        out_dir, new_cfg = gf.compose_concepts(os.path.join(work, 'concepts.json'), a.textenc_iters, a.unet_iters,
                                               os.path.join(work, 'base'), os.path.join(work, 'out'), 'bench',
                                               device=device, tokenizer=WordTokenizer(), log=log)
        torch.cuda.synchronize()
        t2 = time.perf_counter()
        stamps.append((t2, 'end'))
        secs = [tb - ta for (ta, _), (tb, _) in zip(stamps[:-1], stamps[1:])] + [t2 - t1]
        if world > 1:                                   # every rank logged the same stages: slowest rank per stage
            t = torch.tensor(secs, dtype=torch.float64, device=dp.collective_device(device))
            dist.all_reduce(t, op=dist.ReduceOp.MAX)
            secs = t.tolist()
        out['stage_seconds'] = {name.strip('-'): round(v, 2) for (_, name), v in zip(stamps[:-1], secs)}
        out['compose_concepts_seconds'] = round(secs[-1], 2)
        if world > 1:
            stages = ('text_encoder', 'cross_kv', 'spatial')
            out['plan'] = {}
            for stage, (shapes, iters, plan) in zip(stages, plans):
                cost = [sum(gf.solve_cost(shapes[n], iters) for n in p) for p in plan]
                out['plan'][stage] = {'layers': [len(p) for p in plan],
                                      'cost_share': [round(c / max(1, sum(cost)), 4) for c in cost]}
        out['new_concept_tokens'] = sum(len(v['concept_token_ids']) for v in new_cfg.values())
        if rank == 0:
            check_fused(a, out_dir, out)
    finally:
        if world > 1:
            dist.barrier()
            dist.destroy_process_group()
        if rank == 0:
            shutil.rmtree(work, ignore_errors=True)
    if rank == 0:
        print(json.dumps(out))


def write_workload(a, work, out):
    """the synthetic base model directory, the concept checkpoints and concepts.json under `work`"""
    from mixofshow.models.unet_b200 import UNet2DConditionModel
    from mixofshow.utils import model_io
    from transformers import CLIPTextConfig, CLIPTextModel
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
    csd = clip.state_dict()
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
        if a.text_where == 'CLIPEncoderLayer':
            gm = torch.Generator().manual_seed(1050 + c)
            for i in range(12):
                for fc in ('fc1', 'fc2'):
                    m = f'text_model.encoder.layers.{i}.mlp.{fc}'
                    tlora[m + '.lora_down.weight'], tlora[m + '.lora_up.weight'] = _lora_pair(gm, csd[m + '.weight'])
        ulora = (whole_block_unet_lora(sd, cfg, seed=10 + c) if a.unet_where == 'Transformer2DModel'
                 else bench.random_unet_lora(sd, cfg, seed=10 + c))
        params = {'new_concept_embedding': {w: torch.randn(16, 768, generator=g) * 0.02 for w in words},
                  'text_encoder': tlora, 'unet': ulora}
        path = os.path.join(work, f'concept{c}.pth')
        torch.save({'params': params}, path)
        cfgs.append({'lora_path': path, 'unet_alpha': 1.0, 'text_encoder_alpha': 1.0, 'concept_name': ' '.join(words)})
    cfg_path = os.path.join(work, 'concepts.json')
    json.dump(cfgs, open(cfg_path, 'w'))
    del unet, clip, csd
    out['setup_seconds'] = round(time.perf_counter() - t0, 2)


def check_fused(a, out_dir, out):
    """the fused directory must load again (from_pretrained layout) and carry finite weights"""
    import hashlib
    from mixofshow.utils import model_io
    sd, _, _, _, _ = bench.build_workload(a.tiny)
    fused = model_io.load_unet(out_dir)
    h = hashlib.sha256()
    for k, v in sorted(fused.state_dict().items()):
        h.update(k.encode())
        h.update(v.detach().float().contiguous().numpy().tobytes())
    out['fused_unet_sha256'] = h.hexdigest()[:16]
    w = fused.state_dict()['down_blocks.0.attentions.0.transformer_blocks.0.attn2.to_k.weight']
    out['fused_reload_ok'] = bool(torch.isfinite(w).all())
    d0 = sd['down_blocks.0.attentions.0.transformer_blocks.0.attn2.to_k.weight']
    out['example_crosskv_delta_rel'] = round(((w.float().cpu() - d0).norm() / d0.norm()).item(), 5)
    if a.unet_where == 'Transformer2DModel':
        k = 'mid_block.attentions.0.transformer_blocks.0.ff.net.2.weight'
        w = fused.state_dict()[k].float().cpu()
        out['example_ff2_delta_rel'] = round(((w - sd[k]).norm() / sd[k].norm()).item(), 5)
        out['fused_reload_ok'] = out['fused_reload_ok'] and bool(torch.isfinite(w).all())
    out['data'] = 'synthetic (random-init weights, random LoRAs up ~ N(0, 0.02^2), whitespace tokenizer stub)'


if __name__ == '__main__':
    main()
