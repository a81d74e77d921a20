"""The fused model directory as a whole pipeline, and the image the regional CLI writes, on the host:

  * compose_concepts on a synthetic base (tests/synth.py) with and without `vae/` and `scheduler/`: the fused directory
    holds unet/, text_encoder/, tokenizer/, new_concept_cfg.json and a byte-identical copy of each of the two folders the
    base has, nothing else; under two gloo ranks rank 0 alone writes it and the copies are the same bytes;
  * `image_record` (the PNG name and the `.txt` lines) against the reference's own script, run on the argument sets of
    tests/golden/regional_record.json (recipe: tests/golden/make_regional_record_golden.py);
  * `build_model` takes the model's scheduler config, and refuses one the fused step does not compute before loading
    anything;
  * `_sample` with a stand-in pipeline: what each rank writes, with and without a VAE."""
import filecmp
import hashlib
import json
import os
import shutil
import socket
import sys
from types import SimpleNamespace

import pytest
import torch
import torch.multiprocessing as mp

from synth import make_pretrained_dir

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, 'mix-of-show_b200')
TESTS = os.path.join(ROOT, 'tests')
GOLDEN = os.path.join(TESTS, 'golden', 'regional_record.json')

# an SD1.5 `scheduler/scheduler_config.json` (a PNDM config, as the SD1.5 checkpoints ship it) with other betas
SCHEDULER_CFG = {'_class_name': 'PNDMScheduler', '_diffusers_version': '0.6.0', 'beta_end': 0.015,
                 'beta_schedule': 'scaled_linear', 'beta_start': 0.001, 'num_train_timesteps': 1000,
                 'set_alpha_to_one': False, 'skip_prk_steps': True, 'steps_offset': 1, 'trained_betas': None,
                 'clip_sample': False}
FUSED = ['new_concept_cfg.json', 'text_encoder', 'tokenizer', 'unet']


def _write_scheduler(base, cfg=None):
    os.makedirs(os.path.join(base, 'scheduler'), exist_ok=True)
    with open(os.path.join(base, 'scheduler', 'scheduler_config.json'), 'w') as f:
        json.dump(cfg or SCHEDULER_CFG, f, indent=2)


@pytest.fixture(scope='module')
def full_base(tmp_path_factory):
    """a synthetic base with vae/ and scheduler/, and two embedding-only concept checkpoints (no LoRA: the fusion stages
    are not reached, only the orchestration and the save run)"""
    tmp = tmp_path_factory.mktemp('fused_outputs')
    base = make_pretrained_dir(str(tmp / 'base'), clip_layers=1)
    _write_scheduler(base)
    cfgs = []
    for c, name in enumerate(('<cat1> <cat2>', '<dog1>')):
        g = torch.Generator().manual_seed(c)
        path = str(tmp / f'c{c}.pth')
        torch.save({'params': {'new_concept_embedding': {w: torch.randn(16, 768, generator=g) for w in name.split()}}},
                   path)
        cfgs.append({'lora_path': path, 'unet_alpha': 1.0, 'text_encoder_alpha': 1.0, 'concept_name': name})
    cfg_path = str(tmp / 'concepts.json')
    json.dump(cfgs, open(cfg_path, 'w'))
    return tmp, base, cfg_path


def _variant(tmp, base, with_vae, with_scheduler):
    """the full base with the folders it should lack removed"""
    path = str(tmp / f'base_v{int(with_vae)}_s{int(with_scheduler)}')
    if not os.path.isdir(path):
        shutil.copytree(base, path)
        for sub, keep in (('vae', with_vae), ('scheduler', with_scheduler)):
            if not keep:
                shutil.rmtree(os.path.join(path, sub))
    return path


def _same_tree(a, b):
    """every file under a and b, same relative names, same bytes"""
    def files(root):
        return sorted(os.path.relpath(os.path.join(d, f), root) for d, _, fs in os.walk(root) for f in fs)
    names = files(a)
    assert names == files(b) and names
    _, mismatch, errors = filecmp.cmpfiles(a, b, names, shallow=False)
    assert not mismatch and not errors, (mismatch, errors)


@pytest.mark.parametrize('with_vae,with_scheduler', [(True, True), (True, False), (False, True), (False, False)])
def test_fused_directory_contents(full_base, with_vae, with_scheduler):
    import gradient_fusion as gf
    tmp, base, cfg_path = full_base
    base = _variant(tmp, base, with_vae, with_scheduler)
    save = str(tmp / f'out_v{int(with_vae)}_s{int(with_scheduler)}')
    out_dir, new_cfg = gf.compose_concepts(cfg_path, 5, 3, base, save, 'base', device='cpu', log=lambda *a: None)
    assert list(new_cfg) == ['<cat1>', '<cat2>', '<dog1>']
    copied = [sub for sub, present in (('scheduler', with_scheduler), ('vae', with_vae)) if present]
    assert sorted(os.listdir(out_dir)) == sorted(FUSED + copied)
    for sub in copied:
        _same_tree(os.path.join(base, sub), os.path.join(out_dir, sub))


# ------------------------------------------------------------------------------------------------ two gloo ranks
def _free_port():
    with socket.socket() as s:
        s.bind(('127.0.0.1', 0))
        return s.getsockname()[1]


def _compose_worker(rank, world, port, base, cfg_path, save, q):
    import torch.distributed as dist
    sys.path[:0] = [ROOT, PKG, TESTS]
    os.environ.update(MASTER_ADDR='127.0.0.1', MASTER_PORT=str(port))
    dist.init_process_group('gloo', rank=rank, world_size=world)
    try:
        import gradient_fusion as gf
        from mixofshow.utils import model_io
        saved = []
        save_combined = model_io.save_combined_model

        def save_and_note(out_dir, *a, **k):
            saved.append(out_dir)
            return save_combined(out_dir, *a, **k)

        model_io.save_combined_model = save_and_note
        gf.compose_concepts(cfg_path, 5, 3, base, save, 'base', device='cpu', log=lambda *a: None)
        q.put((rank, 'ok', saved))
    except Exception:
        import traceback
        q.put((rank, 'raised', traceback.format_exc()))
    finally:
        dist.destroy_process_group()


def test_two_ranks_write_the_same_copies_once(full_base):
    tmp, base, cfg_path = full_base
    save = str(tmp / 'out_world2')
    ctx = mp.get_context('spawn')
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_compose_worker, args=(r, 2, port, base, cfg_path, save, q)) for r in range(2)]
    try:
        for p in procs:
            p.start()
        res = sorted([q.get(timeout=300) for _ in range(2)], key=lambda t: t[0])
        for p in procs:
            p.join(timeout=60)
            assert p.exitcode == 0
    finally:
        for p in procs:
            if p.is_alive():
                p.kill()
                p.join()
    assert [r[1] for r in res] == ['ok', 'ok'], res
    out_dir = os.path.join(save, 'combined_model_base')
    assert res[0][2] == [out_dir] and res[1][2] == []
    assert sorted(os.listdir(out_dir)) == sorted(FUSED + ['scheduler', 'vae'])
    for sub in ('vae', 'scheduler'):
        _same_tree(os.path.join(base, sub), os.path.join(out_dir, sub))


# ------------------------------------------------------------------------------------------------ the image record
def _golden():
    with open(GOLDEN, encoding='utf-8') as f:
        return json.load(f)


def test_golden_covers_the_cases():
    """no suffix and no condition; a suffix with one condition (and an empty one); both conditions with per-region
    adaptor weight strings and a non-ASCII prompt"""
    cases = _golden()
    assert sorted(cases) == ['both', 'keypose', 'plain', 'sketch']
    assert '------' in cases['plain']['name'] and 'condition: None' in cases['plain']['txt']
    assert '---baseline---' in cases['keypose']['name'] and 'sketch_condition: \n' in cases['keypose']['txt']
    assert 'region_sketch_adaptor_weight: [' in cases['both']['txt'] and 'region_keypose_adaptor_weight: [' in \
        cases['both']['txt'] and 'é' in cases['both']['name']


@pytest.mark.parametrize('tag', ['plain', 'keypose', 'both', 'sketch'])
def test_image_record_matches_the_reference(tag):
    import regionally_controlable_sampling as rcs
    case = _golden()[tag]
    args = rcs.parse_args(case['argv'])
    context_prompt, _ = rcs.prepare_text(args.prompt, args.prompt_rewrite, args.height, args.width)
    lines, name = rcs.image_record(args, context_prompt)
    assert ''.join(lines) == case['txt']
    assert name == case['name']
    assert name.endswith(hashlib.sha256(case['txt'].encode('utf-8')).hexdigest()[:8] + '.png')


# ------------------------------------------------------------------------------------------------ build_model
def _fused_like(tmp_path, with_vae=False):
    base = make_pretrained_dir(str(tmp_path / 'model'), clip_layers=1, with_vae=with_vae)
    json.dump({}, open(os.path.join(base, 'new_concept_cfg.json'), 'w'))
    return base


def _coefficients(scheduler, steps=50):
    scheduler.set_timesteps(steps)
    return [scheduler.coefficients(i) for i in range(steps)]


def test_build_model_takes_the_scheduler_config(tmp_path):
    import regionally_controlable_sampling as rcs
    from mos_b200.scheduler import DPMSolverPP2M
    base = _fused_like(tmp_path, with_vae=True)
    pipe = rcs.build_model(base, device='cpu')
    # the VAE is attached, and the latent grid stays at 1/8 of the image although this VAE upsamples 2x only
    assert pipe.vae is not None and pipe.vae_scale_factor == 8
    assert rcs.build_model(base, device='cpu', with_vae=False).vae is None
    default = _coefficients(DPMSolverPP2M())
    assert _coefficients(pipe.scheduler) == default                          # no scheduler/: the SD1.5 defaults
    _write_scheduler(base)
    got = _coefficients(rcs.build_model(base, device='cpu').scheduler)
    assert got == _coefficients(DPMSolverPP2M.from_pretrained(base, subfolder='scheduler'))
    assert got != default                                                    # the config's betas were read


def test_build_model_refuses_a_scheduler_before_loading(tmp_path, monkeypatch):
    import regionally_controlable_sampling as rcs
    from mixofshow.utils import model_io
    base = _fused_like(tmp_path)
    _write_scheduler(base, dict(SCHEDULER_CFG, prediction_type='v_prediction'))
    loaded = []
    monkeypatch.setattr(model_io, 'load_unet', lambda *a, **k: loaded.append(a))
    with pytest.raises(ValueError, match='prediction_type'):
        rcs.build_model(base, device='cpu')
    assert loaded == []


# ------------------------------------------------------------------------------------------------ what _sample writes
class _VAE:
    config = SimpleNamespace(block_out_channels=(128, 256))

    def decode(self, z):
        return SimpleNamespace(sample=torch.tanh(z[:, :3]).repeat_interleave(2, 2).repeat_interleave(2, 3))


class _Pipe:
    def __init__(self, vae):
        self.vae, self.calls = vae, []

    def __call__(self, **kw):
        self.calls.append(kw)
        lat = torch.randn(1, 4, kw['height'] // 8, kw['width'] // 8, generator=kw['generator'])
        return SimpleNamespace(images=lat)


@pytest.mark.parametrize('rank,model_has_vae', [(0, True), (0, False), (1, True)])
def test_sample_writes(tmp_path, monkeypatch, rank, model_has_vae):
    """rank 0 writes the latents and config.json, and with a VAE the PNG and its .txt under seed_<seed>/; rank 1 loads no
    VAE and writes nothing"""
    import numpy as np
    from PIL import Image
    import regionally_controlable_sampling as rcs
    built = []

    def build(path, device, with_vae=True):
        built.append(with_vae)
        return _Pipe(_VAE() if with_vae and model_has_vae else None)

    monkeypatch.setattr(rcs, 'build_model', build)
    save = str(tmp_path / 'out')
    args = rcs.parse_args(['--pretrained_model', 'fused', '--height', '64', '--width', '128', '--prompt', 'two pets',
                           '--prompt_rewrite', '[a cat]-*-[]-*-[0, 0, 64, 64]', '--seed', '3', '--suffix', 's',
                           '--save_dir', save])
    lat = rcs._sample(args, {}, rank, torch.device('cpu'), None)
    assert built == [rank == 0]
    if rank == 1:
        assert not os.path.exists(save)
        return
    files = sorted(os.path.relpath(os.path.join(d, f), save) for d, _, fs in os.walk(save) for f in fs)
    lines, name = rcs.image_record(args, 'two pets')
    want = ['config.json', 'latents---3---s.pt']
    if model_has_vae:
        want += [name, name[:-4] + '.txt']
    assert files == sorted(want)
    assert torch.equal(torch.load(os.path.join(save, 'latents---3---s.pt'))['latents'], lat)
    if model_has_vae:
        assert name.startswith(os.path.join('seed_3', 'two_pets---s---'))
        assert open(os.path.join(save, name[:-4] + '.txt')).read() == ''.join(lines)
        img = np.asarray(Image.open(os.path.join(save, name)))
        want_img = ((torch.tanh(lat[0, :3] / 0.18215) / 2 + 0.5).clamp(0, 1) * 255).round().to(torch.uint8)
        want_img = want_img.repeat_interleave(2, 1).repeat_interleave(2, 2).permute(1, 2, 0).numpy()
        assert img.shape == (16, 32, 3) and (img == want_img).all()
