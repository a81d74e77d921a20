"""Gradient fusion sharded across ranks on the GPU:

  * each fusion stage called with `solve_names` returns exactly those weights, bit-identical to the full call;
  * `gradient_fusion.main` at world sizes 1, 2 and 3 (spawned ranks sharing the one GPU over gloo) writes bit-identical
    fused models for both LoRA placement pairs, and each rank solves and records exactly what the plan gives it."""
import json
import os
import random
import socket
import sys

import pytest
import torch
import torch.multiprocessing as mp

from synth import make_pretrained_dir

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, 'mix-of-show_b200')
TESTS = os.path.join(ROOT, 'tests')


def _bits(t):
    t = t.detach().cpu().contiguous()
    return t.view(torch.int32) if t.dtype == torch.float32 else t.view(torch.int16)


def _assert_subset_bit_identical(full, part, subset):
    assert sorted(part) == sorted(subset)
    for n in subset:
        assert part[n].shape == full[n].shape, n
        assert torch.equal(_bits(part[n]), _bits(full[n])), n


def _subset(names, seed):
    names = sorted(names)
    return random.Random(seed).sample(names, max(1, len(names) // 3))


def test_stage_subsets_bit_identical_to_the_full_call(cuda):
    import gradient_fusion as gf
    from transformers import CLIPTextConfig, CLIPTextModel
    from oracle import inject
    from oracle import unet as ou
    # ---- spatial (whole-block placement: attention projections, ff.net, proj_in / proj_out)
    u0 = ou.build_unet(0, ou.TINY)
    sd = {k: v.clone() for k, v in u0.state_dict().items()}
    loras = [inject.random_lora_state(u0, seed=10 + c, where='Transformer2DModel', up_std=0.05) for c in range(2)]
    spatial = [{k: v for k, v in l.items() if 'attn2.to_k' not in k and 'attn2.to_v' not in k} for l in loras]
    crosskv = [{k: v for k, v in l.items() if 'attn2.to_k' in k or 'attn2.to_v' in k} for l in loras]
    embeds = [torch.randn(1, 16, 77, 768, generator=torch.Generator().manual_seed(20 + c)) for c in range(2)]
    kw = dict(latent_hw=(16, 16), num_inference_steps=3, seed=0, block_out=ou.TINY['block_out_channels'], layers=1)
    full = gf.merge_spatial_attention(sd, spatial, [1.0, 0.9], embeds, 5, **kw)
    sub = _subset(full, 1)
    part = gf.merge_spatial_attention(sd, spatial, [1.0, 0.9], embeds, 5, solve_names=sub, **kw)
    assert all(v.is_cuda for v in part.values())
    _assert_subset_bit_identical(full, part, sub)
    assert gf.merge_spatial_attention(sd, spatial, [1.0, 0.9], embeds, 5, solve_names=[], **kw) == {}
    # ---- cross-attention K/V
    names = [(i // 2, n) for i, n in enumerate(sorted({k.replace('.lora_down', '').replace('.lora_up', '')
                                                       for k in crosskv[0]}))]
    g = torch.Generator().manual_seed(3)
    feats = [{i: torch.randn(6, 768, generator=g) for i, _ in names} for _ in range(2)]
    full = gf.merge_kv_in_cross_attention(sd, names, feats, crosskv, [1.0, 0.9], 10)
    sub = _subset(full, 2)
    _assert_subset_bit_identical(full, gf.merge_kv_in_cross_attention(sd, names, feats, crosskv, [1.0, 0.9], 10,
                                                                      solve_names=sub), sub)
    # ---- text encoder (CLIPEncoderLayer placement)
    torch.manual_seed(0)
    clip = CLIPTextModel(CLIPTextConfig(vocab_size=1000, hidden_size=768, intermediate_size=3072, num_hidden_layers=2,
                                        num_attention_heads=12, max_position_embeddings=77, eos_token_id=999,
                                        bos_token_id=998, pad_token_id=999)).eval()
    tsd = clip.state_dict()
    tl = [inject.random_lora_state(clip, seed=c, where='CLIPEncoderLayer', up_std=0.05) for c in range(2)]
    g = torch.Generator().manual_seed(9)
    ids = [[torch.cat([torch.tensor([998]), torch.randint(0, 990, (n,), generator=g), torch.tensor([999])])
            for n in (5, 2, 5, 2)] for _ in range(2)]
    full = gf.merge_text_encoder(tsd, tl, [1.0, 0.8], ids, 10, pad_id=999)
    sub = _subset(full, 3)
    _assert_subset_bit_identical(full, gf.merge_text_encoder(tsd, tl, [1.0, 0.8], ids, 10, pad_id=999, solve_names=sub),
                                 sub)


# ------------------------------------------------------------------------------------------------ main() at world 1 / 2 / 3
def _free_port():
    with socket.socket() as s:
        s.bind(('127.0.0.1', 0))
        return s.getsockname()[1]


def _fuse_worker(rank, world, port, argv, q):
    """one torchrun-style rank of `gradient_fusion.main`, noting the plans it computed, the layers it solved, the problems
    it passed to the native solver and the record keys it accumulated"""
    os.environ.update(WORLD_SIZE=str(world), RANK=str(rank), LOCAL_RANK=str(rank), LOCAL_WORLD_SIZE=str(world),
                      MASTER_ADDR='127.0.0.1', MASTER_PORT=str(port))
    sys.path[:0] = [ROOT, PKG, TESTS]
    try:
        import gradient_fusion as gf
        from mos_b200 import ops
        plans, solved, problems, recorded = [], [], [0], {'gram': set(), 'rows': set()}
        fusion_plan, solve_all, solve_batch = gf.fusion_plan, gf.solve_all, ops.lbfgs_solve_batch
        gram_call, rows_call = gf.GramRecorder.__call__, gf._RowRecorder.__call__

        def plan_and_note(shapes, iters, w):
            plans.append(fusion_plan(shapes, iters, w))
            return plans[-1]

        def solve_and_note(jobs, iters, **kw):
            solved.extend(j[0] for j in jobs)
            return solve_all(jobs, iters, **kw)

        def batch_and_note(batch, iters, **kw):
            problems[0] += len(batch)
            return solve_batch(batch, iters, **kw)

        def gram_and_note(self, key, *a):
            gram_call(self, key, *a)
            recorded['gram'].update(self.G)

        def rows_and_note(self, key, *a):
            rows_call(self, key, *a)
            recorded['rows'].update(self.X)

        gf.fusion_plan, gf.solve_all, ops.lbfgs_solve_batch = plan_and_note, solve_and_note, batch_and_note
        gf.GramRecorder.__call__, gf._RowRecorder.__call__ = gram_and_note, rows_and_note
        out_dir, _ = gf.main(argv)
        q.put((rank, 'ok', out_dir, plans, sorted(solved), problems[0], {k: sorted(v) for k, v in recorded.items()}))
    except Exception as exc:
        import traceback
        q.put((rank, 'raised', traceback.format_exc()))


def _run_main(world, argv):
    ctx = mp.get_context('spawn')
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_fuse_worker, args=(r, world, port, argv, q)) for r in range(world)]
    try:
        for p in procs:
            p.start()
        res = sorted([q.get(timeout=900) for _ in range(world)], key=lambda t: t[0])
        for p in procs:
            p.join(timeout=120)
            assert p.exitcode == 0
        return res
    finally:
        for p in procs:
            if p.is_alive():
                p.kill()
                p.join()


def _concepts(tmp_path, base, unet_where, text_where):
    from transformers import CLIPTextModel
    from oracle import inject
    from oracle import unet as ou
    ref_unet = ou.build_unet(0, ou.TINY)
    clip = CLIPTextModel.from_pretrained(os.path.join(base, 'text_encoder'))
    cfgs = []
    for c, name in enumerate(('<cat1> <cat2>', '<dog1>', '<hat1>')):
        g = torch.Generator().manual_seed(c)
        params = {'new_concept_embedding': {w: torch.randn(16, 768, generator=g) * 0.02 for w in name.split()},
                  'text_encoder': inject.random_lora_state(clip, seed=c, where=text_where, up_std=0.05),
                  'unet': inject.random_lora_state(ref_unet, seed=10 + c, where=unet_where, up_std=0.05)}
        path = str(tmp_path / f'c{c}.pth')
        torch.save({'params': params}, path)
        cfgs.append({'lora_path': path, 'unet_alpha': 1.0 - 0.1 * c, 'text_encoder_alpha': 0.9 + 0.05 * c,
                     'concept_name': name})
    cfg_path = str(tmp_path / 'concepts.json')
    json.dump(cfgs, open(cfg_path, 'w'))
    return cfg_path


def _files(out_dir, sub):
    folder = os.path.join(out_dir, sub)
    return sorted(os.listdir(folder)), folder


@pytest.mark.parametrize('where', [('Attention', 'CLIPAttention'), ('Transformer2DModel', 'CLIPEncoderLayer')],
                         ids=lambda w: w[0])
def test_main_sharded_over_ranks_is_bit_identical_to_one_rank(cuda, tmp_path, where):
    from safetensors.torch import load_file
    import gradient_fusion as gf
    base = make_pretrained_dir(str(tmp_path / 'base'))
    cfg_path = _concepts(tmp_path, base, *where)
    outs = {}
    for world in (1, 2, 3):
        argv = ['--concept_cfg', cfg_path, '--save_path', str(tmp_path / f'w{world}'), '--pretrained_models', base,
                '--optimize_textenc_iters', '8', '--optimize_unet_iters', '3', '--suffix', 'mr']
        res = _run_main(world, argv)
        assert [r[1] for r in res] == ['ok'] * world, [r[2] for r in res if r[1] != 'ok']
        outs[world] = res
        if world == 1:
            everything = set(res[0][4])
            continue
        plans = res[0][3]
        assert len(plans) == 3 and all(r[3] == plans for r in res)          # text, cross-K/V, spatial: same plan everywhere
        owned = set()
        for rank, _, _, _, solved, problems, recorded in res:
            mine = [n for p in plans for n in p[rank]]
            assert solved == sorted(mine) and problems == len(mine)
            owned |= set(mine)
            assert recorded['rows'] == sorted({gf.record_key(n) for n in plans[0][rank]})
            assert recorded['gram'] == sorted({gf.record_key(n) for n in plans[2][rank]})
            print(f'world {world} rank {rank}: {len(mine)} layers ({[len(p[rank]) for p in plans]} per stage)')
        assert owned == everything
    ref = outs[1][0][2]
    for world in (2, 3):
        out = outs[world][0][2]
        for sub in ('unet', 'text_encoder'):
            names, folder = _files(out, sub)
            assert names == _files(ref, sub)[0]
            for f in names:
                if f.endswith('.safetensors'):
                    a, b = load_file(os.path.join(folder, f)), load_file(os.path.join(ref, sub, f))
                    assert sorted(a) == sorted(b)
                    for k in a:
                        assert a[k].dtype == b[k].dtype and torch.equal(_bits(a[k]), _bits(b[k])), (world, k)
        assert open(os.path.join(out, 'new_concept_cfg.json')).read() == open(os.path.join(ref, 'new_concept_cfg.json')).read()
        names, folder = _files(out, 'tokenizer')
        assert names == _files(ref, 'tokenizer')[0]
        for f in names:
            assert open(os.path.join(folder, f), 'rb').read() == open(os.path.join(ref, 'tokenizer', f), 'rb').read(), f
