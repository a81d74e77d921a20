"""CFG-split sampling, host side, on CPU with gloo at world size 2: the argument checks of `cfg_group` in all three
pipelines and the entry script (raised on both ranks, before any text encoding, and leaving no rank waiting), and the
eps exchange itself (group-rank order, the initial-latents broadcast).  The split loop on the GPU is covered by
tests/test_cfg_split_gpu.py."""
import os
import socket
import sys

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, 'mix-of-show_b200')


def _free_port():
    with socket.socket() as s:
        s.bind(('127.0.0.1', 0))
        return s.getsockname()[1]


class _NoTextEncoder:
    """a text encoder that counts its calls: the refusals must come before any of them"""
    calls = 0

    def __call__(self, *a, **k):
        _NoTextEncoder.calls += 1
        raise AssertionError('text encoding ran before the cfg_group checks')


def _pipes():
    from mixofshow.models.unet_b200 import UNet2DConditionModel
    from mixofshow.pipelines.pipeline_edlora import EDLoRAPipeline, StableDiffusionPipeline
    from mixofshow.pipelines.pipeline_regionally_t2iadapter import RegionallyT2IAdapterPipeline
    out = {}
    for name, cls in (('edlora', EDLoRAPipeline), ('sd', StableDiffusionPipeline),
                      ('regional', RegionallyT2IAdapterPipeline)):
        unet = UNet2DConditionModel(block_out_channels=(32, 64), layers_per_block=1)
        pipe = cls(unet=unet, text_encoder=_NoTextEncoder(), tokenizer=lambda *a, **k: None)
        if hasattr(pipe, 'set_new_concept_cfg'):
            pipe.set_new_concept_cfg({})
        out[name] = pipe
    return out


def _call(name, pipe, **kw):
    if name == 'regional':
        return pipe(prompt=[('a photo', [('a cat', None, [0, 0, 1, 0.5])])], height=64, width=64, **kw)
    return pipe(prompt='a photo', height=64, width=64, **kw)


def _refusals(rank):
    from mixofshow.utils.ptp_util import AttentionStore
    pipes = _pipes()
    one = [dist.new_group([0]), dist.new_group([1])][rank]      # every rank creates every group
    msgs = []
    for name, pipe in pipes.items():
        for kw in ({'cfg_group': one}, {'cfg_group': dist.group.WORLD, 'guidance_scale': 1.0},
                   {'cfg_group': dist.group.WORLD, 'guidance_scale': 0.5}):
            with pytest.raises(ValueError) as e:
                _call(name, pipe, **kw)
            msgs.append((name, str(e.value)))
    pipes['edlora'].set_controller(AttentionStore())
    with pytest.raises(ValueError) as e:
        _call('edlora', pipes['edlora'], cfg_group=dist.group.WORLD)
    msgs.append(('edlora', str(e.value)))
    return msgs


def _exchange(rank):
    from mos_b200.dp import CFGExchange
    ex = CFGExchange(dist.group.WORLD, (1, 4, 3, 5), 'cpu')
    half = torch.full((1, 4, 3, 5), float(rank + 1))
    out = ex.all_gather(half).clone()
    lat = torch.randn(1, 4, 3, 5, generator=torch.Generator().manual_seed(10 + rank))
    ex.broadcast(lat)
    return ex.half, ex.bytes_per_step, out, lat


def _worker(rank, world, port, job, q):
    sys.path[:0] = [ROOT, PKG]
    os.environ.update(MASTER_ADDR='127.0.0.1', MASTER_PORT=str(port))
    try:
        dist.init_process_group('gloo', rank=rank, world_size=world)
        res = {'refusals': _refusals, 'exchange': _exchange}[job](rank)
        dist.barrier()                  # both ranks get here: nobody is left inside a collective
        q.put((rank, 'ok', res))
        dist.destroy_process_group()
    except Exception:
        import traceback
        q.put((rank, 'raised', traceback.format_exc()))


def _run(job, world=2):
    ctx = mp.get_context('spawn')
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, world, port, job, q)) for r in range(world)]
    try:
        for p in procs:
            p.start()
        res = sorted([q.get(timeout=300) for _ in range(world)], key=lambda t: t[0])
        for p in procs:
            p.join(timeout=60)
            assert p.exitcode == 0
        assert [r[1] for r in res] == ['ok'] * world, [r[2] for r in res if r[1] != 'ok']
        return [r[2] for r in res]
    finally:
        for p in procs:
            if p.is_alive():
                p.kill()
                p.join()


def test_refusals_on_both_ranks_before_text_encoding():
    msgs = _run('refusals')
    assert msgs[0] == msgs[1]
    assert len(msgs[0]) == 3 * 3 + 1
    for name, m in msgs[0]:
        assert 'cfg_group' in m, (name, m)
    by_kind = [m for _, m in msgs[0]]
    assert all('exactly two ranks' in m for m in by_kind[0:9:3])
    assert all('guidance_scale' in m for i, m in enumerate(by_kind[:9]) if i % 3)
    assert 'attention controller' in by_kind[9]


def test_exchange_gathers_in_group_rank_order_and_broadcasts_rank0():
    (h0, b0, out0, lat0), (h1, b1, out1, lat1) = _run('exchange')
    assert (h0, h1) == (0, 1) and b0 == b1 == 2 * 4 * 3 * 5 * 4
    want = torch.cat([torch.full((1, 4, 3, 5), 1.0), torch.full((1, 4, 3, 5), 2.0)])
    assert torch.equal(out0, want) and torch.equal(out1, want)
    assert torch.equal(lat0, lat1)
    assert torch.equal(lat0, torch.randn(1, 4, 3, 5, generator=torch.Generator().manual_seed(10)))


def test_refusal_without_a_process_group():
    sys.path[:0] = [ROOT, PKG]
    from mos_b200 import dp
    assert not dist.is_initialized()
    dp.check_cfg_group(None, 1.0)           # no group: nothing to check, whatever the guidance
    with pytest.raises(ValueError, match='initialised'):
        dp.check_cfg_group(object(), 7.5)


@pytest.mark.parametrize('world', ['3', '4'])
def test_entry_script_refuses_other_world_sizes(monkeypatch, world):
    import regionally_controlable_sampling as rcs
    monkeypatch.setenv('WORLD_SIZE', world)
    with pytest.raises(ValueError, match='1 process, or on 2 under torchrun'):
        rcs.main(['--pretrained_model', 'x'])
    assert not dist.is_initialized()
