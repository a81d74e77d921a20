"""The fused model directory sampled as a whole pipeline, and the image the regional CLI writes, on the GPU.  The synthetic
base (tests/synth.py) carries the tiny VAE of oracle/vae.py (one 2x level); images are compared with the fp32 oracle
decode of the same latents within 2 of 255 levels, the tolerance of tests/test_vae_gpu.py::test_pipeline_decodes_to_pil.

  * two concepts fused on a base with vae/ give a directory whose `EDLoRAPipeline.from_pretrained(...)(prompt).images[0]`
    is a PIL image, the oracle decode of that call's latents;
  * the regional CLI, with key-pose and sketch condition images, writes `seed_<seed>/<prompt>---<suffix>---<hash8>.png`
    and its `.txt`; the PNG is the oracle decode of the saved latents, and the latents are bit for bit those of the same
    command on the same directory without vae/ (the VAE does not change the latent grid: build_model);
  * the same command on two ranks: rank 0 alone loads the VAE and writes one PNG, the same bits as a one-process decode of
    its latents;
  * a 1024 x 2048 image (the `_2x` conditions of regionally_sample.sh) decoded through the CLI by an SD1.5-size VAE."""
import hashlib
import json
import os
import shutil
import socket
import sys

import numpy as np
import pytest
import torch
import torch.multiprocessing as mp

from synth import make_pretrained_dir

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, 'mix-of-show_b200')
TESTS = os.path.join(ROOT, 'tests')
COND = os.path.join(TESTS, 'golden', 't2i_conditions')
POSE, SKETCH = os.path.join(COND, 'harry+catA+dogA_pose.png'), os.path.join(COND, 'harry+catA+dogA_sketch.png')
REWRITE = '[a cat]-*-[blurry]-*-[10,20,500,480]|[a dog]-*-[blurry]-*-[20,540,500,1000]'


def _pixels(path):
    from PIL import Image
    return torch.from_numpy(np.asarray(Image.open(path)).astype('float32'))


def _oracle_pixels(vae_dir, latents):
    """the fp32 oracle decode of `latents` with the weights of `vae_dir`, as 8-bit levels [H, W, 3]"""
    from safetensors.torch import load_file
    from oracle import vae as ov
    ref = ov.build_vae(0, ov.TINY_VAE)
    ref.load_state_dict(load_file(os.path.join(vae_dir, 'diffusion_pytorch_model.safetensors')))
    with torch.no_grad():
        dec = ref.decode(latents.float().cpu() / 0.18215)
    return ((dec / 2 + 0.5).clamp(0, 1)[0].permute(1, 2, 0) * 255).round()


def _files(root):
    return sorted(os.path.relpath(os.path.join(d, f), root) for d, _, fs in os.walk(root) for f in fs)


def _same_tree(a, b):
    assert _files(a) == _files(b) and _files(a)
    for f in _files(a):
        assert open(os.path.join(a, f), 'rb').read() == open(os.path.join(b, f), 'rb').read(), f


# ------------------------------------------------------------------------------------------------ fused directory
def test_fused_directory_samples_a_pil_image(cuda, tmp_path):
    import gradient_fusion
    from PIL import Image
    from transformers import CLIPTextModel
    from mixofshow.pipelines.pipeline_edlora import EDLoRAPipeline
    from oracle import inject
    from oracle import unet as ou
    base = make_pretrained_dir(str(tmp_path / 'base'))
    clip = CLIPTextModel.from_pretrained(os.path.join(base, 'text_encoder'))
    cfgs = []
    for c, name in enumerate(('<cat1> <cat2>', '<dog1>')):
        g = torch.Generator().manual_seed(c)
        params = {'new_concept_embedding': {w: torch.randn(16, 768, generator=g) * 0.02 for w in name.split()},
                  'text_encoder': inject.random_lora_state(clip, seed=c, where='CLIPAttention', up_std=0.05),
                  'unet': inject.random_lora_state(ou.build_unet(0, ou.TINY), seed=10 + c, up_std=0.05)}
        torch.save({'params': params}, str(tmp_path / f'c{c}.pth'))
        cfgs.append({'lora_path': str(tmp_path / f'c{c}.pth'), 'unet_alpha': 1.0, 'text_encoder_alpha': 1.0,
                     'concept_name': name})
    json.dump(cfgs, open(str(tmp_path / 'concepts.json'), 'w'))
    out_dir, _ = gradient_fusion.main(['--concept_cfg', str(tmp_path / 'concepts.json'), '--save_path',
                                       str(tmp_path / 'fused'), '--pretrained_models', base,
                                       '--optimize_textenc_iters', '8', '--optimize_unet_iters', '3', '--suffix', 'img'])
    _same_tree(os.path.join(base, 'vae'), os.path.join(out_dir, 'vae'))
    pipe = EDLoRAPipeline.from_pretrained(out_dir)
    kw = dict(negative_prompt='blurry', height=64, width=64, num_inference_steps=4, guidance_scale=7.5)
    prompt = 'a <cat1> <cat2> next to a <dog1>'
    img = pipe(prompt, generator=torch.Generator().manual_seed(3), **kw).images[0]
    lat = pipe(prompt, generator=torch.Generator().manual_seed(3), output_type='latent', **kw).images
    assert isinstance(img, Image.Image) and img.size == (64, 64)          # the tiny VAE upsamples a 32 x 32 latent 2x
    got = torch.from_numpy(np.asarray(img).astype('float32'))
    err = (got - _oracle_pixels(os.path.join(out_dir, 'vae'), lat)).abs().max().item()
    print(f'fused directory, pipe(prompt).images[0] vs oracle decode of its latents: max {err} levels')
    assert err <= 2.0


# ------------------------------------------------------------------------------------------------ regional CLI
def _regional_base(tmp_path):
    from mixofshow.utils import model_io
    from oracle import adapter as oa
    base = make_pretrained_dir(str(tmp_path / 'base'))
    json.dump({}, open(os.path.join(base, 'new_concept_cfg.json'), 'w'))
    adapters = {}
    for kind, cin in (('keypose', 3), ('sketch', 1)):
        adapters[kind] = str(tmp_path / f'{kind}_adapter')
        model_io.save_t2i_adapter(oa.build_adapter(30 + cin, dict(in_channels=cin, **oa.TINY_ADAPTER)), adapters[kind])
    return base, adapters


def _argv(base, adapters, save):
    return ['--pretrained_model', base, '--num_inference_steps', '3', '--prompt', 'two animals in the snow',
            '--negative_prompt', 'blurry', '--seed', '7', '--suffix', 'e2e', '--prompt_rewrite', REWRITE,
            '--keypose_condition', POSE, '--keypose_adapter', adapters['keypose'], '--keypose_adaptor_weight', '0.8',
            '--region_keypose_adaptor_weight', '[0, 0, 512, 480]-0.5',
            '--sketch_condition', SKETCH, '--sketch_adapter', adapters['sketch'], '--sketch_adaptor_weight', '0.6',
            '--region_sketch_adaptor_weight', '[20, 540, 500, 1000]-1.2', '--save_dir', save]


def _expected(base):
    """the .txt text and PNG name of _argv's command, written out"""
    txt = (f'pretrained_model: {base}\ncontext_prompt: two animals in the snow\nneg_context_prompt: blurry\n'
           f'sketch_condition: {SKETCH}\nsketch_adaptor_weight: 0.6\nregion_sketch_adaptor_weight: [20, 540, 500, 1000]-1.2\n'
           f'keypose_condition: {POSE}\nkeypose_adaptor_weight: 0.8\nregion_keypose_adaptor_weight: [0, 0, 512, 480]-0.5\n'
           f'random seed: 7\nprompt_rewrite: {REWRITE}\n')
    name = os.path.join('seed_7', f'two_animals_in_the_snow---e2e---{hashlib.sha256(txt.encode()).hexdigest()[:8]}')
    return txt, name


def test_regional_cli_writes_the_image(cuda, tmp_path):
    import regionally_controlable_sampling as rcs
    base, adapters = _regional_base(tmp_path)
    txt, name = _expected(base)
    save = str(tmp_path / 'with_vae')
    lat = rcs.main(_argv(base, adapters, save))
    assert tuple(lat.shape) == (1, 4, 64, 128)                          # 512 x 1024 conditions, a 1/8 latent grid
    assert _files(save) == sorted(['config.json', 'latents---7---e2e.pt', name + '.png', name + '.txt'])
    assert open(os.path.join(save, name + '.txt')).read() == txt
    saved = torch.load(os.path.join(save, 'latents---7---e2e.pt'))
    got = _pixels(os.path.join(save, name + '.png'))
    assert got.shape == (128, 256, 3)                                    # the tiny VAE upsamples 2x
    err = (got - _oracle_pixels(os.path.join(base, 'vae'), saved['latents'])).abs().max().item()
    print(f'regional CLI PNG vs oracle decode of the saved latents: max {err} levels')
    assert err <= 2.0
    # ---- the same command on the same directory without vae/: the latents file alone, the same latents
    shutil.move(os.path.join(base, 'vae'), str(tmp_path / 'vae_off'))
    save2 = str(tmp_path / 'without_vae')
    rcs.main(_argv(base, adapters, save2))
    assert _files(save2) == ['config.json', 'latents---7---e2e.pt']
    plain = torch.load(os.path.join(save2, 'latents---7---e2e.pt'))
    assert torch.equal(plain['latents'].view(torch.int32), saved['latents'].view(torch.int32))
    assert {k: v for k, v in plain['config'].items() if k != 'save_dir'} == \
        {k: v for k, v in saved['config'].items() if k != 'save_dir'}


def _free_port():
    with socket.socket() as s:
        s.bind(('127.0.0.1', 0))
        return s.getsockname()[1]


def _cli_worker(rank, world, port, argv, q):
    """one torchrun-style rank of regionally_controlable_sampling.main, noting the files it writes and its VAE loads"""
    os.environ.update(WORLD_SIZE=str(world), RANK=str(rank), LOCAL_RANK=str(rank), LOCAL_WORLD_SIZE=str(world),
                      MASTER_ADDR='127.0.0.1', MASTER_PORT=str(port))
    sys.path[:0] = [ROOT, PKG, TESTS]
    try:
        from PIL import Image
        import regionally_controlable_sampling as rcs
        from mixofshow.utils import model_io
        written, vae_loads = [], []
        save, img_save, load_vae = torch.save, Image.Image.save, model_io.load_vae

        def save_and_note(obj, path, *a, **k):
            written.append(str(path))
            return save(obj, path, *a, **k)

        def img_save_and_note(self, path, *a, **k):
            written.append(str(path))
            return img_save(self, path, *a, **k)

        def open_and_note(path, mode='r', *a, **k):
            if any(c in mode for c in 'wax+'):
                written.append(str(path))
            return open(path, mode, *a, **k)

        def load_vae_and_note(*a, **k):
            vae_loads.append(a)
            return load_vae(*a, **k)

        torch.save, Image.Image.save, rcs.open, model_io.load_vae = \
            save_and_note, img_save_and_note, open_and_note, load_vae_and_note
        lat = rcs.main(argv)
        q.put((rank, 'ok', {'latents': lat.cpu().numpy(), 'written': written, 'vae_loads': len(vae_loads)}))
    except Exception:
        import traceback
        q.put((rank, 'raised', traceback.format_exc()))


def _run_two_ranks(argv):
    ctx = mp.get_context('spawn')
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_cli_worker, args=(r, 2, port, argv, q)) for r in range(2)]
    try:
        for p in procs:
            p.start()
        res = sorted([q.get(timeout=900) for _ in range(2)], key=lambda t: t[0])
        for p in procs:
            p.join(timeout=120)
            assert p.exitcode == 0
        assert [r[1] for r in res] == ['ok', 'ok'], [r[2] for r in res if r[1] != 'ok']
        return [r[2] for r in res]
    finally:
        for p in procs:
            if p.is_alive():
                p.kill()
                p.join()


def test_regional_cli_two_ranks_one_image(cuda, tmp_path):
    import regionally_controlable_sampling as rcs
    from mixofshow.pipelines.pipeline_edlora import decode_latents
    from mixofshow.utils import model_io
    base, adapters = _regional_base(tmp_path)
    _, name = _expected(base)
    save = str(tmp_path / 'split')
    r0, r1 = _run_two_ranks(_argv(base, adapters, save))
    assert r1['written'] == [] and r1['vae_loads'] == 0 and r0['vae_loads'] == 1
    want = sorted(['config.json', 'latents---7---e2e.pt', name + '.png', name + '.txt'])
    assert sorted(os.path.relpath(p, save) for p in r0['written']) == want and _files(save) == want
    assert np.array_equal(r0['latents'].view(np.int32), r1['latents'].view(np.int32))
    split = _pixels(os.path.join(save, name + '.png'))
    # rank 0's decode is a one-process decode: given the same latents, the same bits
    vae = model_io.load_vae(base)
    one = decode_latents(vae, torch.from_numpy(r0['latents']).cuda())[0]
    assert torch.equal(split, torch.from_numpy(np.asarray(one).astype('float32')))
    # against the one-process command: the split latents may differ in the last bits (a CFG half at batch 1 can take
    # other split-K counts, DESIGN.md §6), and so may the pixels, each image staying within 2 levels of the oracle decode
    # of its own latents.  Measured on an H100 80GB HBM3: latents 2.2e-3 rel-L2 apart after the 3 steps, PNGs at most 1
    # level apart (mean 0.09)
    single_save = str(tmp_path / 'single')
    single = rcs.main(_argv(base, adapters, single_save))
    same_latents = np.array_equal(single.cpu().numpy().view(np.int32), r0['latents'].view(np.int32))
    single_px = _pixels(os.path.join(single_save, name + '.png'))
    d = (split - single_px).abs()
    lat_err = (torch.from_numpy(r0['latents']) - single.cpu()).norm().item() / single.norm().item()
    print(f'two ranks vs one process: latents bit-identical {same_latents} (rel-L2 {lat_err:.3e}); PNG pixels differ '
          f'by max {d.max().item()} / mean {d.mean().item():.4f} levels')
    if same_latents:
        assert torch.equal(split, single_px)
    else:
        assert lat_err < 5e-3
        for px, lat in ((split, torch.from_numpy(r0['latents'])), (single_px, single.cpu())):
            assert (px - _oracle_pixels(os.path.join(base, 'vae'), lat)).abs().max().item() <= 2.0


def test_regional_cli_decodes_1024x2048(cuda, tmp_path):
    """one 128 x 256 latent decoded through the CLI by an SD1.5-size VAE (83.65 M parameters): 32768 mid-block tokens"""
    import regionally_controlable_sampling as rcs
    from mixofshow.models.vae_b200 import AutoencoderKL
    from mixofshow.utils import model_io
    from oracle import vae as ov
    base = make_pretrained_dir(str(tmp_path / 'base'), with_vae=False)
    model_io.save_vae(AutoencoderKL({k: v.detach() for k, v in ov.build_vae(0).state_dict().items()}, device='cpu'), base)
    json.dump({}, open(os.path.join(base, 'new_concept_cfg.json'), 'w'))
    save = str(tmp_path / 'out')
    lat = rcs.main(['--pretrained_model', base, '--height', '1024', '--width', '2048', '--num_inference_steps', '2',
                    '--prompt', 'three people near the castle', '--seed', '19', '--save_dir', save, '--prompt_rewrite',
                    '[a man]-*-[]-*-[4, 6, 1024, 490]|[a girl]-*-[]-*-[14, 490, 1024, 920]|[a giant]-*-[]-*-[2, 1302, 1024, 1992]'])
    assert tuple(lat.shape) == (1, 4, 128, 256) and torch.isfinite(lat).all()
    pngs = [f for f in _files(save) if f.endswith('.png')]
    assert len(pngs) == 1 and pngs[0].startswith(os.path.join('seed_19', 'three_people_near_the_castle------'))
    px = _pixels(os.path.join(save, pngs[0]))
    assert px.shape == (1024, 2048, 3) and px.std().item() > 0
    assert os.path.exists(os.path.join(save, pngs[0][:-4] + '.txt'))
