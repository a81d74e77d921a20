"""The T2I-Adapter on the GPU (mos_b200/adapter_engine.py behind mixofshow/models/adapter_b200.py) against the fp32 oracle
(oracle/adapter.py, run on the GPU with TF32 off), the regional pipeline and entry script driven by the condition images of
tests/golden/t2i_conditions, and every adapter launch under the GEMM launch audit and tests/adapter_audit.py.

Tolerances (rel-L2): features <= 5e-3 (fp16 operands through 10 convolutions); pipeline latents after 3 CFG steps
<= 5e-3, the target of test_regional_gpu.py::test_regional_pipeline_call_vs_oracle_loop.
"""
import json
import os

import numpy as np
import pytest
import torch

import adapter_audit as aa
import gemm_audit as ga
from test_regional_gpu import _b200_unet, _fractions, _math_sdpa, _oracle_spatial_weight, rel_l2

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
POSE = os.path.join(HERE, 'golden', 't2i_conditions', 'harry+catA+dogA_pose.png')
SKETCH = os.path.join(HERE, 'golden', 't2i_conditions', 'harry+catA+dogA_sketch.png')

# every launch of both adapters at 512 x 1024 (adapter_engine.py): conv_in and block1 through the implicit 3x3 conv,
# in_conv as a plain GEMM, block2 with the resnet add fetched through shared memory; the unshuffle, ReLU and pooling
GEMM_KEYS = {'rows|tma|fp16|conv', 'rows|tma|fp16', 'rows+res_smem|tma|fp16'}
ADAPTER_KEYS = {'pixel_unshuffle|fp16', 'relu_rows|fp16', 'avgpool2x|fp16'}


def _image(path, mode):
    """condition PNG -> fp32 NCHW [1, C, H, W] in [0, 1] (same size: no resampling)"""
    from PIL import Image
    a = np.asarray(Image.open(path).convert(mode), dtype=np.float32) / 255.0
    a = a[:, :, None] if a.ndim == 2 else a
    return torch.from_numpy(a.transpose(2, 0, 1).copy())[None]


@pytest.mark.parametrize('cin', [3, 1])
def test_features_full_size_vs_oracle(cuda, cin):
    """SD adapter widths (320, 640, 1280, 1280), 2 resnets per level, at 768 x 1536 (config 4)"""
    from mixofshow.models.adapter_b200 import T2IAdapter
    from oracle import adapter as oa
    ref = oa.build_adapter(cin, dict(in_channels=cin))
    ad = T2IAdapter(ref.state_dict(), in_channels=cin)
    img = torch.rand(1, cin, 768, 1536, generator=torch.Generator().manual_seed(10 + cin))
    feats = ad(img.cuda())
    eng = ad._engine(1, 768, 1536)
    with torch.no_grad():
        want = ref.cuda()(img.cuda())
    assert len(feats) == 4 and eng.launches == 31
    errs = [rel_l2(f, w) for f, w in zip(feats, want)]
    print(f'T2I-Adapter Cin={cin} 768x1536 features vs fp32 oracle: rel-L2 ' + ', '.join(f'{e:.2e}' for e in errs))
    for f, w, e in zip(feats, want, errs):
        assert f.shape == w.shape and f.dtype == torch.float32 and e <= 5e-3


def _tiny_pipe(tmp_path):
    """tiny 2-level UNet (oracle.unet.TINY) with a 2-level key-pose / sketch adapter pair saved and loaded through
    from_pretrained; -> (pipe, oracle UNet, oracle adapters)"""
    from mixofshow.models.adapter_b200 import T2IAdapter
    from mixofshow.pipelines.pipeline_regionally_t2iadapter import RegionallyT2IAdapterPipeline
    from mixofshow.utils import model_io
    from oracle import adapter as oa
    from oracle import inject
    from oracle import unet as ou
    ref = ou.build_unet(0, ou.TINY)
    inject.install_region_processors(ref)
    pipe = RegionallyT2IAdapterPipeline(unet=_b200_unet(ref, ou.TINY)).to('cuda')
    pipe.set_new_concept_cfg({})
    oracle = {}
    for kind, cin in (('keypose', 3), ('sketch', 1)):
        oracle[kind] = oa.build_adapter(20 + cin, dict(in_channels=cin, **oa.TINY_ADAPTER))
        model_io.save_t2i_adapter(oracle[kind], str(tmp_path / kind))
        setattr(pipe, f'{kind}_adapter', T2IAdapter.from_pretrained(str(tmp_path / kind)))
    return pipe, ref, oracle


HEIGHT, WIDTH = 512, 1024
BOXES = _fractions([[0, 10, 512, 340], [5, 340, 512, 690], [2, 690, 512, 1020]], HEIGHT, WIDTH)
SPEC = '[0,40,512,340]-0.3|[16,690,500,1000]-1.5'


def _call(pipe, steps, lat, ehs, regs, **kw):
    return pipe(prompt_embeds=ehs.cuda(), region_list=[(r.cuda(), b) for r, b in regs], latents=lat.clone(),
                height=HEIGHT, width=WIDTH, num_inference_steps=steps, guidance_scale=7.5, output_type='latent',
                keypose_adaptor_weight=0.8, sketch_adaptor_weight=0.5, region_sketch_adaptor_weight=SPEC, **kw).images


def _inputs():
    g = lambda s: torch.Generator().manual_seed(s)                        # noqa: E731
    lat = torch.randn(1, 4, HEIGHT // 8, WIDTH // 8, generator=g(3))
    ehs = torch.randn(2, 16, 77, 768, generator=g(4))
    regs = [(torch.randn(2, 16, 77, 768, generator=g(5 + i)), BOXES[i]) for i in range(3)]
    return lat, ehs, regs


def test_pipeline_from_condition_images_vs_oracle_loop(cuda, tmp_path):
    """RegionallyT2IAdapterPipeline.__call__ with the two fixture PNGs (RGBA 1024 x 512, converted as the reference script
    does), 3 regions, a region_sketch_adaptor_weight string, 3 DPM-Solver++ steps at CFG 7.5, against the oracle adapters +
    the restated adapter mixing + the oracle UNet loop"""
    from PIL import Image
    from oracle import edlora_ref as er
    from oracle.schedulers import DPMSolverMultistepScheduler
    pipe, ref, oracle = _tiny_pipe(tmp_path)
    lat, ehs, regs = _inputs()
    pose, sketch = Image.open(POSE).convert('RGB'), Image.open(SKETCH).convert('L')
    steps = 3
    res = _call(pipe, steps, lat, ehs, regs, keypose_adapter_input=[pose], sketch_adapter_input=[sketch])
    with torch.no_grad():
        kp = oracle['keypose'].cuda()(_image(POSE, 'RGB').cuda())
        sk = oracle['sketch'].cuda()(_image(SKETCH, 'L').cuda())
    adapter = [torch.cat([_oracle_spatial_weight(kp[i].cpu(), 0.8, '', HEIGHT, WIDTH)
                          + _oracle_spatial_weight(sk[i].cpu(), 0.5, SPEC, HEIGHT, WIDTH)] * 2).cuda() for i in range(2)]
    sched = DPMSolverMultistepScheduler()
    sched.set_timesteps(steps)
    ref = ref.cuda()
    x = lat.clone()
    kw = {'region_list': [(r.cuda(), b) for r, b in regs], 'height': HEIGHT, 'width': WIDTH}
    for t in sched.timesteps:
        with torch.no_grad(), _math_sdpa():
            eps = ref(torch.cat([x, x]).cuda(), torch.tensor([int(t), int(t)]).cuda(), ehs.cuda(),
                      cross_attention_kwargs=kw, down_block_additional_residuals=[a.clone() for a in adapter]).sample.cpu()
        x = sched.step(er.cfg_combine(eps, 7.5), int(t), x).prev_sample
    e = rel_l2(res, x)
    print(f'pipeline from condition images (2 adapters, 3 regions, weight string) vs oracle loop: rel-L2 {e:.3e}')
    assert e <= 5e-3
    # the image path is the state path with the adapters' own outputs
    from mixofshow.pipelines.pipeline_regionally_t2iadapter import preprocess_adapter_image
    kst = pipe.keypose_adapter(preprocess_adapter_image([pose], HEIGHT, WIDTH).cuda())
    sst = pipe.sketch_adapter(preprocess_adapter_image([sketch], HEIGHT, WIDTH).cuda())
    res_state = _call(pipe, steps, lat, ehs, regs, keypose_adapter_state=kst, sketch_adapter_state=sst)
    assert torch.equal(res_state, res)
    # the conditions must matter
    res_none = _call(pipe, steps, lat, ehs, regs)
    assert rel_l2(res_none, res) > 1e-3


def test_adapter_runs_once_per_call(cuda, tmp_path):
    """a 6-step call runs each adapter engine once (reference :474-482: before the loop)"""
    from PIL import Image
    pipe, _, _ = _tiny_pipe(tmp_path)
    lat, ehs, regs = _inputs()
    calls = {}
    for kind in ('keypose', 'sketch'):
        eng = getattr(pipe, f'{kind}_adapter')._engine(1, HEIGHT, WIDTH)
        fwd = eng.forward

        def counted(x, _fwd=fwd, _kind=kind):
            calls[_kind] = calls.get(_kind, 0) + 1
            return _fwd(x)
        eng.forward = counted
    res = _call(pipe, 6, lat, ehs, regs, keypose_adapter_input=Image.open(POSE).convert('RGB'),
                sketch_adapter_input=Image.open(SKETCH).convert('L'))
    assert calls == {'keypose': 1, 'sketch': 1} and torch.isfinite(res).all()


def test_entry_script_with_condition_images(cuda, tmp_path):
    """regionally_controlable_sampling.main with --keypose_condition / --sketch_condition and local adapter directories on
    the synthetic model directory: the latent size follows the images, and the conditions change the result"""
    import regionally_controlable_sampling as rcs
    from mixofshow.utils import model_io
    from oracle import adapter as oa
    from synth import make_pretrained_dir
    base = make_pretrained_dir(str(tmp_path / 'base'), with_vae=False)
    json.dump({}, open(os.path.join(base, 'new_concept_cfg.json'), 'w'))
    dirs = {}
    for kind, cin in (('keypose', 3), ('sketch', 1)):
        dirs[kind] = str(tmp_path / f'{kind}_adapter')
        model_io.save_t2i_adapter(oa.build_adapter(30 + cin, dict(in_channels=cin, **oa.TINY_ADAPTER)), dirs[kind],
                                  safe_serialization=kind == 'keypose')
    common = ['--pretrained_model', base, '--num_inference_steps', '3', '--prompt', 'two animals', '--seed', '7',
              '--prompt_rewrite', '[a cat]-*-[blurry]-*-[10,20,500,480]|[a dog]-*-[blurry]-*-[20,540,500,1000]']
    save = str(tmp_path / 'out')
    lat = rcs.main(common + ['--keypose_condition', POSE, '--keypose_adapter', dirs['keypose'],
                             '--sketch_condition', SKETCH, '--sketch_adapter', dirs['sketch'], '--save_dir', save])
    assert tuple(lat.shape) == (1, 4, 64, 128) and torch.isfinite(lat).all()
    plain = rcs.main(common + ['--height', '512', '--width', '1024'])
    assert rel_l2(plain, lat) > 1e-3
    cfg = json.load(open(os.path.join(save, 'config.json')))
    assert cfg['keypose_condition'] == POSE and cfg['sketch_condition'] == SKETCH
    assert cfg['keypose_adapter'] == dirs['keypose'] and (cfg['height'], cfg['width']) == (512, 1024)
    assert os.path.exists(os.path.join(save, 'latents---7.pt'))


def _adapters_512x1024(audit):
    """AdapterEngine with the SD adapter widths at 512 x 1024: the key-pose (3 input channels) and the sketch (1) adapter,
    each forward run inside `audit()`, a zero-argument callable that returns a recorder"""
    from mos_b200.adapter_engine import AdapterEngine
    from oracle import adapter as oa
    for seed, cin in ((0, 3), (1, 1)):
        ref = oa.build_adapter(seed, dict(in_channels=cin))
        eng = AdapterEngine({k: v.detach().clone() for k, v in ref.state_dict().items()}, 1, 512, 1024, in_channels=cin)
        img = torch.rand(1, cin, 512, 1024, generator=torch.Generator().manual_seed(seed)).cuda()
        with audit():
            eng.forward(img)
            torch.cuda.synchronize()


def test_launch_audits(cuda):
    """every launch of both SD-width adapters at 512 x 1024 under the GEMM and the adapter launch audits"""
    gstats, astats = ga.Stats(), aa.Stats()
    _adapters_512x1024(lambda: ga.Recorder(gstats))
    _adapters_512x1024(lambda: aa.Recorder(astats))
    print(gstats.table())
    print(astats.table())
    assert not gstats.failures, '\n'.join(gstats.failures[:20])
    assert not astats.failures, '\n'.join(astats.failures[:20])
    assert set(gstats.rows) == GEMM_KEYS and set(astats.rows) == ADAPTER_KEYS, (sorted(gstats.rows), sorted(astats.rows))
    assert sum(r['n'] for r in gstats.rows.values()) == 2 * 19 and sum(r['n'] for r in astats.rows.values()) == 2 * 12
