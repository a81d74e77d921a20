"""Gradient fusion across ranks, CPU only: the layer partition plan (gradient_fusion.fusion_plan) and the sharded
orchestration of compose_concepts over gloo, with the three fusion stages replaced by stubs (their GPU arithmetic, and its
bit-identity under sharding, is tests/test_fusion_multirank_gpu.py)."""
import hashlib
import json
import os
import random
import socket
import subprocess
import sys

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, 'mix-of-show_b200')
TESTS = os.path.join(ROOT, 'tests')


def sd15_stage_shapes(unet_where='Transformer2DModel', text_where='CLIPEncoderLayer'):
    """{stage: {weight name: shape}} of an SD1.5 fusion (16 transformer blocks, 12 CLIP layers), by name and shape only"""
    chans = [('down_blocks', b, j, c) for b, c in enumerate((320, 640, 1280)) for j in range(2)]
    chans += [('mid_block', None, 0, 1280)]
    chans += [('up_blocks', b, j, c) for b, c in zip((1, 2, 3), (1280, 640, 320)) for j in range(3)]
    spatial, kv = {}, {}
    for part, b, j, c in chans:
        tn = f'{part}.attentions.{j}' if b is None else f'{part}.{b}.attentions.{j}'
        blk = tn + '.transformer_blocks.0'
        for a in ('attn1.to_q', 'attn1.to_k', 'attn1.to_v', 'attn1.to_out.0', 'attn2.to_q', 'attn2.to_out.0'):
            spatial[f'{blk}.{a}.weight'] = (c, c)
        kv[f'{blk}.attn2.to_k.weight'] = (c, 768)
        kv[f'{blk}.attn2.to_v.weight'] = (c, 768)
        if unet_where == 'Transformer2DModel':
            spatial[f'{blk}.ff.net.0.proj.weight'] = (8 * c, c)
            spatial[f'{blk}.ff.net.2.weight'] = (c, 4 * c)
            spatial[f'{tn}.proj_in.weight'] = (c, c, 1, 1)
            spatial[f'{tn}.proj_out.weight'] = (c, c, 1, 1)
    text = {}
    for i in range(12):
        m = f'text_model.encoder.layers.{i}'
        for p in ('q_proj', 'k_proj', 'v_proj', 'out_proj'):
            text[f'{m}.self_attn.{p}.weight'] = (768, 768)
        if text_where == 'CLIPEncoderLayer':
            text[f'{m}.mlp.fc1.weight'] = (3072, 768)
            text[f'{m}.mlp.fc2.weight'] = (768, 3072)
    return {'text': (text, 500), 'kv': (kv, 500), 'spatial': (spatial, 50)}


PLACEMENTS = [('Attention', 'CLIPAttention'), ('Transformer2DModel', 'CLIPEncoderLayer')]


@pytest.mark.parametrize('where', PLACEMENTS, ids=lambda w: w[0])
@pytest.mark.parametrize('world', [1, 2, 3, 4, 5, 8])
def test_plan_covers_every_weight_once_within_the_greedy_bound(where, world):
    import gradient_fusion as gf
    for stage, (shapes, iters) in sd15_stage_shapes(*where).items():
        plan = gf.fusion_plan(shapes, iters, world)
        assert len(plan) == world
        flat = [n for p in plan for n in p]
        assert sorted(flat) == sorted(shapes) and len(set(flat)) == len(flat), stage
        assert all(p == sorted(p) for p in plan)
        cost = {n: gf.solve_cost(s, iters) for n, s in shapes.items()}
        loads = [sum(cost[n] for n in p) for p in plan]
        # Graham's 4/3 bound of longest-processing-time-first is relative to the optimum, which may exceed this lower bound
        # of it (total / W, largest job); holding against the lower bound is an empirical property of the SD1.5 shapes
        assert 3 * max(loads) <= 4 * max(sum(loads) / world, max(cost.values())), (stage, loads)
        if world == 1:
            assert plan == [sorted(shapes)]


def test_plan_cost_is_the_closure_gemm():
    import gradient_fusion as gf
    assert gf.solve_cost((1280, 5120), 50) == 1280 * 5120 * 5120 * 50
    assert gf.solve_cost((320, 320, 1, 1), 50) == gf.solve_cost((320, 320), 50)


def test_plan_is_independent_of_key_order_and_process():
    import gradient_fusion as gf
    shapes, iters = sd15_stage_shapes()['spatial']
    ref = gf.fusion_plan(shapes, iters, 3)
    rng = random.Random(0)
    for _ in range(5):
        keys = list(shapes)
        rng.shuffle(keys)
        assert gf.fusion_plan({k: shapes[k] for k in keys}, iters, 3) == ref
    # another interpreter with another string-hash seed
    code = ('import json, sys; sys.path[:0] = [%r, %r]; import test_fusion_sharding as t, gradient_fusion as gf; '
            's, i = t.sd15_stage_shapes()["spatial"]; print(json.dumps(gf.fusion_plan(dict(reversed(list(s.items()))), i, 3)))'
            % (PKG, TESTS))
    env = dict(os.environ, PYTHONHASHSEED='12345')
    out = subprocess.run([sys.executable, '-c', code], capture_output=True, text=True, env=env, timeout=300, check=True)
    assert json.loads(out.stdout.strip().splitlines()[-1]) == ref


# ------------------------------------------------------------------------------------------------ compose_concepts on gloo
def _free_port():
    with socket.socket() as s:
        s.bind(('127.0.0.1', 0))
        return s.getsockname()[1]


def _digest(sd):
    return {k: hashlib.sha256(v.detach().float().contiguous().numpy().tobytes()).hexdigest() for k, v in sd.items()}


def _compose_worker(rank, world, port, base, cfg_path, save, fail_stage, q):
    """one rank of compose_concepts with recording stubs for the three stages"""
    sys.path[:0] = [ROOT, PKG, TESTS]
    os.environ['MASTER_ADDR'] = '127.0.0.1'
    os.environ['MASTER_PORT'] = str(port)
    dist.init_process_group('gloo', rank=rank, world_size=world)
    try:
        import gradient_fusion as gf
        from mixofshow.utils import model_io
        from transformers import CLIPTextModel
        from test_fusion_orchestration import WordTokenizer
        made, seen, saved = {}, {}, []
        load_unet, save_combined = model_io.load_unet, model_io.save_combined_model
        model_io.load_unet = lambda *a, **k: made.setdefault('unet', load_unet(*a, **k))
        model_io.load_text_encoder = lambda path, subfolder='text_encoder', **kw: made.setdefault(
            'te', CLIPTextModel.from_pretrained(os.path.join(path, subfolder)).eval())

        def save_and_note(out_dir, *a, **k):
            saved.append(out_dir)
            return save_combined(out_dir, *a, **k)

        model_io.save_combined_model = save_and_note

        def stub(tag, bump):
            def stage(sd, *args, solve_names=None, **kw):
                seen[tag] = list(solve_names)
                if tag == fail_stage and rank == world - 1:
                    raise ValueError(f'{tag}: no closure evaluation gave a finite loss')
                return {n: sd[n].float() * 0.5 + bump for n in solve_names}
            return stage

        gf.merge_text_encoder = stub('text', 1.0)
        gf.merge_kv_in_cross_attention = stub('kv', 2.0)
        gf.merge_spatial_attention = stub('spatial', 3.0)
        gf.compose_concepts(cfg_path, 7, 3, base, save, 'base', device='cpu', tokenizer=WordTokenizer(),
                            log=lambda *a: None)
        q.put((rank, 'ok', seen, saved, _digest(made['unet'].state_dict()), _digest(made['te'].state_dict())))
    except Exception as exc:
        q.put((rank, 'raised', type(exc).__name__, str(exc)))
    finally:
        dist.destroy_process_group()


def _run_world(world, base, cfg_path, save, fail_stage=None):
    ctx = mp.get_context('spawn')
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_compose_worker, args=(r, world, port, base, cfg_path, save, fail_stage, q))
             for r in range(world)]
    try:
        for p in procs:
            p.start()
        res = sorted([q.get(timeout=300) for _ in range(world)], key=lambda t: t[0])
        for p in procs:
            p.join(timeout=60)
            assert p.exitcode == 0
        return res
    finally:
        for p in procs:
            if p.is_alive():
                p.kill()
                p.join()


@pytest.fixture(scope='module')
def concepts(tmp_path_factory):
    """a tiny pretrained directory and two concept checkpoints (as tests/test_fusion_orchestration.py)"""
    from transformers import CLIPTextConfig, CLIPTextModel
    from mixofshow.models.unet_b200 import UNet2DConditionModel
    from mixofshow.utils import model_io
    from oracle import inject
    from oracle import unet as ou
    tmp = tmp_path_factory.mktemp('sharding')
    torch.manual_seed(0)
    unet = UNet2DConditionModel(block_out_channels=ou.TINY['block_out_channels'], layers_per_block=ou.TINY['layers_per_block'])
    base = str(tmp / 'base')
    model_io.save_unet(unet, base)
    clip = CLIPTextModel(CLIPTextConfig(vocab_size=49408, hidden_size=768, intermediate_size=3072, num_hidden_layers=1,
                                        num_attention_heads=12, max_position_embeddings=77)).eval()
    clip.save_pretrained(os.path.join(base, 'text_encoder'))
    ref_unet = ou.build_unet(0, ou.TINY)
    cfgs = []
    for c, name in enumerate(('<cat1> <cat2>', '<dog1>')):
        g = torch.Generator().manual_seed(c)
        params = {'new_concept_embedding': {w: torch.randn(16, 768, generator=g) for w in name.split()},
                  'text_encoder': inject.random_lora_state(clip, seed=c, where='CLIPEncoderLayer'),
                  'unet': inject.random_lora_state(ref_unet, seed=10 + c, where='Transformer2DModel')}
        path = str(tmp / f'c{c}.pth')
        torch.save({'params': params}, path)
        cfgs.append({'lora_path': path, 'unet_alpha': 0.8 + 0.1 * c, 'text_encoder_alpha': 1.0, 'concept_name': name})
    cfg_path = str(tmp / 'concepts.json')
    json.dump(cfgs, open(cfg_path, 'w'))
    import gradient_fusion as gf
    _, te, kv, sp, _ = gf.parse_new_concepts(cfg_path)
    expected = {'text': gf.lora_weight_names(te), 'kv': [n for _, n in gf.cross_kv_layer_names(unet)],
                'spatial': gf.lora_weight_names(sp)}
    return tmp, base, cfg_path, expected


@pytest.mark.parametrize('world', [2, 3])
def test_compose_concepts_sharded_over_gloo(concepts, world):
    """every stage's weights are split over the ranks as the plan says, the exchanged results leave every rank with the
    same models, and only rank 0 writes the fused directory"""
    tmp, base, cfg_path, expected = concepts
    save = str(tmp / f'out{world}')
    res = _run_world(world, base, cfg_path, save)
    assert [r[1] for r in res] == ['ok'] * world, res
    for tag, names in expected.items():
        owned = [set(r[2][tag]) for r in res]
        assert set().union(*owned) == set(names) and sum(map(len, owned)) == len(names), tag
    assert res[0][3] == [os.path.join(save, 'combined_model_base')] and all(r[3] == [] for r in res[1:])
    assert os.listdir(save) == ['combined_model_base']
    for r in res[1:]:
        assert r[4] == res[0][4] and r[5] == res[0][5]
    # the stubs' results reached every rank (0.5 w + bump of the stage that owns w)
    from mixofshow.utils import model_io
    fused, orig = model_io.load_unet(os.path.join(save, 'combined_model_base')), model_io.load_unet(base)
    for tag, bump in (('kv', 2.0), ('spatial', 3.0)):
        for n in expected[tag]:
            want = orig.state_dict()[n].float() * 0.5 + bump
            assert _digest({n: fused.state_dict()[n]}) == _digest({n: want}) == {n: res[-1][4][n]}, n


@pytest.mark.parametrize('world', [2, 3])
def test_a_failing_rank_makes_every_rank_raise(concepts, world):
    tmp, base, cfg_path, _ = concepts
    save = str(tmp / f'fail{world}')
    res = _run_world(world, base, cfg_path, save, fail_stage='kv')
    assert [r[1] for r in res] == ['raised'] * world
    assert res[-1][2] == 'ValueError' and 'finite loss' in res[-1][3]                   # the failing rank's own error
    assert all(r[2] == 'RuntimeError' and 'another rank' in r[3] for r in res[:-1])
    assert not os.path.exists(os.path.join(save, 'combined_model_base'))
