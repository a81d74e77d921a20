"""T2I-Adapter host logic on the CPU: the oracle's parameter names and counts, the diffusers-layout save / load round trip,
the configurations and geometries the GPU path rejects, the condition-image preprocessing, the entry script's condition
options, and the launch-audit rules of the adapter kernels against torch through the norm audit's stand-in library."""
import json
import os

import pytest
import torch
import torch.nn.functional as F

import adapter_audit as aa

HERE = os.path.dirname(os.path.abspath(__file__))
COND = os.path.join(HERE, 'golden', 't2i_conditions')
POSE = os.path.join(COND, 'harry+catA+dogA_pose.png')
SKETCH = os.path.join(COND, 'harry+catA+dogA_sketch.png')
F16 = torch.float16


# ------------------------------------------------------------------------------------------------- network and files
@pytest.mark.parametrize('cin,count', [(3, 77_369_280), (1, 77_000_640)])
def test_oracle_keys_and_parameter_count(cin, count):
    from mos_b200.adapter_engine import adapter_param_shapes
    from oracle import adapter as oa
    ref = oa.build_adapter(0, dict(in_channels=cin))
    sd = ref.state_dict()
    assert sum(v.numel() for v in sd.values()) == count
    assert {k: tuple(v.shape) for k, v in sd.items()} == adapter_param_shapes(cin, (320, 640, 1280, 1280), 2)
    assert 'adapter.conv_in.weight' in sd and 'adapter.body.1.in_conv.weight' in sd
    assert 'adapter.body.0.in_conv.weight' not in sd and 'adapter.body.3.in_conv.weight' not in sd
    assert tuple(sd['adapter.body.3.resnets.1.block2.weight'].shape) == (1280, 1280, 1, 1)


@pytest.mark.parametrize('safe', [True, False])
def test_save_load_round_trip_bit_identical(tmp_path, safe):
    from mixofshow.models.adapter_b200 import T2IAdapter
    from mixofshow.utils import model_io
    from oracle import adapter as oa
    ref = oa.build_adapter(3, dict(in_channels=1, **oa.TINY_ADAPTER))
    model_io.save_t2i_adapter(ref, str(tmp_path), safe_serialization=safe)
    name = 'diffusion_pytorch_model.' + ('safetensors' if safe else 'bin')
    assert sorted(os.listdir(tmp_path)) == sorted(['config.json', name])
    ad = T2IAdapter.from_pretrained(str(tmp_path), device='cpu')
    assert ad.config.in_channels == 1 and ad.config.channels == [320, 640] and ad.config.num_res_blocks == 2
    assert ad.total_downscale_factor == 16 and ad.dtype == torch.float32
    got, want = ad.state_dict(), ref.state_dict()
    assert got.keys() == want.keys()
    for k in want:
        assert got[k].dtype == torch.float32 and torch.equal(got[k], want[k]), k


def _edit_config(path, **kw):
    cfg = json.load(open(os.path.join(path, 'config.json')))
    cfg.update(kw)
    json.dump(cfg, open(os.path.join(path, 'config.json'), 'w'))


@pytest.mark.parametrize('edit', [dict(adapter_type='light_adapter'), dict(adapter_type='full_adapter_xl'),
                                  dict(downscale_factor=16), dict(num_res_blocks=3)])
def test_from_pretrained_rejects_unsupported_config(tmp_path, edit):
    from mixofshow.models.adapter_b200 import T2IAdapter
    from mixofshow.utils import model_io
    from oracle import adapter as oa
    model_io.save_t2i_adapter(oa.build_adapter(0, oa.TINY_ADAPTER), str(tmp_path))
    _edit_config(str(tmp_path), **edit)
    with pytest.raises(ValueError):
        T2IAdapter.from_pretrained(str(tmp_path), device='cpu')


def test_from_pretrained_hub_id_is_not_fetched():
    from mixofshow.models.adapter_b200 import T2IAdapter
    with pytest.raises(ValueError, match='hub ids are not downloaded'):
        T2IAdapter.from_pretrained('TencentARC/t2iadapter_openpose_sd14v1')


@pytest.mark.parametrize('channels', [(320, 640, 1280, 1000), (64, 128), (320, 400)])
def test_engine_rejects_channels_off_the_gemm_tile(channels):
    from mos_b200.adapter_engine import AdapterEngine
    with pytest.raises(ValueError, match='multiple of 160'):
        AdapterEngine({}, 1, 512, 1024, channels=channels, device='cpu')


@pytest.mark.parametrize('hw,channels', [((512, 1000), (320, 640, 1280, 1280)), ((520, 1024), (320, 640, 1280, 1280)),
                                         ((504, 1024), (320, 640)), ((512, 1032), (320, 640, 1280))])
def test_engine_rejects_sizes_that_do_not_tile(hw, channels):
    from mos_b200.adapter_engine import AdapterEngine
    with pytest.raises(ValueError, match='multiples of'):
        AdapterEngine({}, 1, *hw, channels=channels, device='cpu')


# ------------------------------------------------------------------------------------------------- preprocessing
def _restated(img, mode, size):
    """independent statement: PIL convert + resize, pixel bytes read back through tobytes()"""
    from PIL import Image
    im = Image.open(img).convert(mode)
    if size != im.size:
        im = im.resize(size, Image.Resampling.LANCZOS)
    w, h = im.size
    v = torch.frombuffer(bytearray(im.tobytes()), dtype=torch.uint8).double()
    v = v.view(h, w, -1).permute(2, 0, 1)[None]
    return (v / 255.0).float()


@pytest.mark.parametrize('path,mode', [(POSE, 'RGB'), (SKETCH, 'L')])
@pytest.mark.parametrize('height,width', [(512, 1024), (256, 640)])
def test_preprocess_adapter_image_vs_restatement(path, mode, height, width):
    from PIL import Image
    from mixofshow.pipelines.pipeline_regionally_t2iadapter import preprocess_adapter_image
    im = Image.open(path)
    assert im.mode == 'RGBA' and im.size == (1024, 512)
    for arg in (im.convert(mode), [im.convert(mode)]):
        got = preprocess_adapter_image(arg, height, width)
        assert got.dtype == torch.float32 and tuple(got.shape) == (1, 3 if mode == 'RGB' else 1, height, width)
        assert torch.equal(got, _restated(path, mode, (width, height)))
    t = torch.rand(1, 3, 8, 8)
    assert preprocess_adapter_image(t, 512, 1024) is t


# ------------------------------------------------------------------------------------------------- entry script
def test_script_takes_the_size_from_the_conditions(tmp_path):
    import regionally_controlable_sampling as rcs
    args = rcs.parse_args(['--pretrained_model', 'x', '--keypose_condition', POSE, '--keypose_adapter', str(tmp_path),
                           '--sketch_condition', SKETCH, '--sketch_adapter', str(tmp_path)])
    assert (args.height, args.width) == (768, 1536)
    conds = rcs.load_conditions(args)
    assert (args.height, args.width) == (512, 1024)
    assert conds['keypose'].mode == 'RGB' and conds['sketch'].mode == 'L'
    args = rcs.parse_args(['--pretrained_model', 'x'])
    assert rcs.load_conditions(args) == {} and (args.height, args.width) == (768, 1536)


def test_script_rejects_mismatched_conditions(tmp_path):
    from PIL import Image
    import regionally_controlable_sampling as rcs
    small = str(tmp_path / 'small.png')
    Image.open(SKETCH).resize((512, 256)).save(small)
    args = rcs.parse_args(['--pretrained_model', 'x', '--keypose_condition', POSE, '--keypose_adapter', str(tmp_path),
                           '--sketch_condition', small, '--sketch_adapter', str(tmp_path)])
    with pytest.raises(ValueError, match='same size'):
        rcs.load_conditions(args)


@pytest.mark.parametrize('kind', ['keypose', 'sketch'])
def test_script_rejects_condition_without_adapter(kind):
    import regionally_controlable_sampling as rcs
    args = rcs.parse_args(['--pretrained_model', 'x', f'--{kind}_condition', POSE if kind == 'keypose' else SKETCH])
    with pytest.raises(ValueError, match=f'--{kind}_adapter'):
        rcs.load_conditions(args)


# ------------------------------------------------------------------------------------------------- launch audit rules
def rnd(shape, seed, scale=1.0, dtype=torch.float32):
    return (torch.randn(shape, generator=torch.Generator().manual_seed(seed)) * scale).to(dtype)


class StandIn:
    """writes the rounded float64 reference of every adapter entry point into the windows its record reads from the ABI
    arguments; `mut` names one defect to inject after the correct result is written"""

    def __init__(self, mut=None):
        self.mut, self.recorder = mut, None

    def __getattr__(self, name):
        if name not in aa.ENTRY_POINTS:
            raise AttributeError(name)
        return lambda *args: self._launch(name, args)

    def _launch(self, entry, args):
        S = aa._Storages(self.recorder._ctx[0], self.recorder.registered)
        rec = aa.record(entry, aa.abi_of(entry, args[:len(aa._ARGS[entry])]), S, self.recorder._ctx[2])
        refs = aa.reference(dict(rec, **{'in': {k: v.clone() for k, v in rec['in'].items()}}))
        t = rec['targets'][0]
        flat = S.flat(*t['mem'])
        w = flat.as_strided(t['size'], t['stride'], t['off'])
        w.copy_(refs[t['name']][0].to(w.dtype))
        m = self.mut
        if m == 'unshuffle_ij' and entry == 'mos_pixel_unshuffle':         # column c*64 + j*8 + i
            B, Ho, Wo, K = t['size']
            w.copy_(w.clone().view(B, Ho, Wo, K // 64, 8, 8).transpose(4, 5).reshape(B, Ho, Wo, K))
        if m == 'pool_past' and entry == 'mos_avgpool2x':                   # one element past the pooled window
            last = t['off'] + sum((s - 1) * st for s, st in zip(t['size'], t['stride']))
            flat[last + 1] = 1.0
        if m == 'relu_pads' and entry == 'mos_relu_rows':                   # ReLU over the whole pitch
            a = rec['abi']
            rows = flat.as_strided((a['M'], a['ld']), (a['ld'], 1), t['off'])
            rows.copy_(rows.clamp(min=0))
        if m == 'pool_two_ulp' and entry == 'mos_avgpool2x':               # one output two ulps off
            w.view(torch.int16).view(-1)[5] += 2
        return 0


@pytest.fixture
def adapter_audit(monkeypatch):
    """adapter_audit(mut=None) -> an adapter_audit.Recorder over the stand-in library (CPU tensors)"""
    from mos_b200 import _lib, adapter_ops
    monkeypatch.setattr(adapter_ops, 'current_stream', lambda: None)

    def make(mut=None):
        lib = StandIn(mut)
        monkeypatch.setattr(_lib, 'lib', lambda: lib)
        r = aa.Recorder()
        lib.recorder = r
        return r
    return make


def ok(r):
    assert not r.stats.failures, '\n'.join(r.stats.failures)
    return r


def flagged(r, letter):
    assert any(f'({letter})' in e for e in r.stats.failures), r.stats.failures


def run_adapter_kernels(make, mut=None, dtype=F16, B=2, Cin=3, H=32, W=48, C=320):
    from mos_b200 import adapter_ops
    img = torch.rand(B, Cin, H, W, generator=torch.Generator().manual_seed(1))
    K = 64 * Cin
    y = torch.full((B * (H // 8) * (W // 8), K + 16), 7.0, dtype=dtype)           # pitched rows: pad columns untouched
    t = rnd((B * 6 * 8, C + 32), 2, 2.0, dtype)                                   # pitched: the pad columns hold negatives
    t0 = t.clone()
    x = rnd((B * 6 * 8, C), 3, 2.0, dtype)
    p = torch.zeros(B * 3 * 4 + 1, C, dtype=dtype)                                 # one spare row past the window
    with make(mut) as r:
        adapter_ops.pixel_unshuffle(img, y)
        adapter_ops.relu_rows(t, M=B * 6 * 8, C=C)
        adapter_ops.avgpool2x(x, p, B=B, H=6, W=8, C=C)
    return r, dict(img=img, y=y, t0=t0, t=t, x=x, p=p)


@pytest.mark.parametrize('dtype', [F16, torch.bfloat16])
def test_adapter_kernel_references_vs_torch(adapter_audit, dtype):
    r, o = run_adapter_kernels(adapter_audit, dtype=dtype)
    ok(r)
    dt = 'fp16' if dtype == F16 else 'bf16'
    assert set(r.stats.rows) == {f'pixel_unshuffle|{dt}', f'relu_rows|{dt}', f'avgpool2x|{dt}'}
    B, K, C = 2, 192, 320
    want = F.pixel_unshuffle(o['img'], 8).permute(0, 2, 3, 1).reshape(-1, K).to(dtype)
    assert torch.equal(o['y'][:, :K], want) and (o['y'][:, K:] == 7).all()
    assert torch.equal(o['t'][:, :C], F.relu(o['t0'][:, :C])) and torch.equal(o['t'][:, C:], o['t0'][:, C:])
    x = o['x'].double().view(B, 6, 8, C).permute(0, 3, 1, 2)
    pool = F.avg_pool2d(x, 2).permute(0, 2, 3, 1).reshape(-1, C)
    assert torch.allclose(o['p'][:-1].double(), pool, rtol=2 ** -7, atol=1e-6) and (o['p'][-1] == 0).all()


@pytest.mark.parametrize('mut,letter', [('unshuffle_ij', 'a'), ('pool_past', 'c'), ('relu_pads', 'c'),
                                        ('pool_two_ulp', 'a')])
def test_adapter_kernel_mutations_flagged(adapter_audit, mut, letter):
    r, _ = run_adapter_kernels(adapter_audit, mut)
    flagged(r, letter)


def test_unshuffle_of_a_pitched_image_flagged(adapter_audit):
    from mos_b200 import adapter_ops
    img = torch.rand(1, 3, 16, 24)[:, :, :, :16]
    with adapter_audit() as r:
        adapter_ops.pixel_unshuffle(img, torch.zeros(4, 192, dtype=F16))
    flagged(r, 'p')


def test_pool_with_pitched_input_read_at_the_wrong_pitch_flagged(adapter_audit):
    from mos_b200 import adapter_ops
    x = rnd((2 * 6 * 8, 336), 4, dtype=F16)[:, :320]
    with adapter_audit() as r:
        adapter_ops.avgpool2x(x, torch.zeros(2 * 3 * 4, 320, dtype=F16), B=2, H=6, W=8, C=320, ldx=320)
    flagged(r, 'p')
