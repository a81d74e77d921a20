"""Image sizes that are multiples of 8 pixels but not of 64 (latent sides that do not halve exactly three times): the
level sizes the UNet works at, the nearest-resize index rule of its up blocks, the regional pipeline's refusal of sizes
whose levels its region rule misreads, and the float64 launch-audit references of the two resampling kernels at odd
extents.  CPU only; the GPU side is tests/test_image_sizes_gpu.py.

diffusers' UNet2DConditionModel samples at any latent size: Downsample2D (3x3, stride 2, pad 1) gives ceil(h / 2), and
when a latent side is not a multiple of 2^(levels - 1) (`forward_upsample_size`) every non-final up block interpolates
(nearest, explicit size) to the size of the skip it is concatenated with.
"""
import random

import pytest
import torch
import torch.nn.functional as F

import norm_audit as na

# latent sizes: every level odd in both sides (520 x 392), even then odd (528 x 528), odd on top and exact below
# (1000 x 1000), a one-pixel-wide strip, and the exact-halving sizes the suite already samples at
LATENTS = [(65, 49), (66, 66), (125, 125), (8, 1), (72, 72), (64, 64), (96, 192), (33, 33), (128, 256)]
CHAINS = {(65, 49): [(65, 49), (33, 25), (17, 13), (9, 7)],
          (66, 66): [(66, 66), (33, 33), (17, 17), (9, 9)],
          (125, 125): [(125, 125), (63, 63), (32, 32), (16, 16)],
          (8, 1): [(8, 1), (4, 1), (2, 1), (1, 1)],
          (72, 72): [(72, 72), (36, 36), (18, 18), (9, 9)]}
SMALL = dict(block_out_channels=(320, 320, 320, 320), layers_per_block=1)     # SD1.5's 4 levels, narrow and shallow


def test_level_sizes_rule():
    from mos_b200.engine import level_sizes
    for (h, w), chain in CHAINS.items():
        assert level_sizes(h, w, 4) == chain
    assert level_sizes(64, 64, 4) == [(64, 64), (32, 32), (16, 16), (8, 8)]
    assert level_sizes(33, 33, 2) == [(33, 33), (17, 17)]


def _trace_oracle(cfg, h, w, seed=0):
    """run the oracle UNet at latent h x w; returns (output shape, downsampler output sizes, upsampler output sizes,
    the input sizes of every up-block resnet)"""
    from oracle import unet as ou
    unet = ou.build_unet(seed, cfg)
    down, up, res_in = [], [], []
    hooks = []
    for name, m in unet.named_modules():
        cn = m.__class__.__name__
        if cn == 'Downsample2D':
            hooks.append(m.register_forward_hook(lambda m, i, o: down.append(tuple(o.shape[2:]))))
        elif cn == 'Upsample2D':
            hooks.append(m.register_forward_hook(lambda m, i, o: up.append(tuple(o.shape[2:]))))
        elif cn == 'ResnetBlock2D' and name.startswith('up_blocks'):
            hooks.append(m.register_forward_hook(lambda m, i, o: res_in.append(tuple(i[0].shape[2:]))))
    g = torch.Generator().manual_seed(seed + 1)
    x = torch.randn(1, 4, h, w, generator=g)
    ehs = torch.randn(1, 77, 768, generator=g)
    with torch.no_grad():
        out = unet(x, torch.tensor([500]), ehs).sample
    for hk in hooks:
        hk.remove()
    return tuple(out.shape), down, up, res_in


@pytest.mark.parametrize('h,w', [(65, 49), (66, 66), (125, 125), (8, 1)])
def test_oracle_goes_through_diffusers_level_sizes(h, w):
    """The SD1.5-topology oracle samples at these latents (it used to raise on the concat of a 2x-upsampled level with an
    odd skip) and passes through the level sizes diffusers gives: ceil on the way down, the next skip's size on the way
    up."""
    shape, down, up, res_in = _trace_oracle(SMALL, h, w)
    chain = CHAINS[(h, w)]
    assert shape == (1, 4, h, w)
    assert down == chain[1:]
    assert up == list(reversed(chain[:-1]))
    want = [s for s in reversed(chain) for _ in range(2)]                     # 2 resnets per up block
    assert res_in == want


def test_oracle_tiny_at_odd_latent():
    """TINY (two levels) at a 33 x 33 latent: 33 -> 17 and back to 33"""
    from oracle import unet as ou
    shape, down, up, _ = _trace_oracle(ou.TINY, 33, 33)
    assert shape == (1, 4, 33, 33) and down == [(17, 17)] and up == [(33, 33)]


def test_oracle_unchanged_at_exact_sizes():
    """At a latent that halves exactly, the explicit-size path the oracle now has is never taken: its output equals the
    scale-factor-2 upsampling bit for bit (nearest at exactly 2x is dst >> 1 either way)"""
    from oracle import unet as ou
    unet = ou.build_unet(0, SMALL)
    g = torch.Generator().manual_seed(5)
    x, ehs = torch.randn(1, 4, 16, 24, generator=g), torch.randn(1, 77, 768, generator=g)
    with torch.no_grad():
        a = unet(x, torch.tensor([500]), ehs).sample
        for blk in unet.up_blocks[:-1]:
            up = blk.upsamplers[0]
            up.forward = (lambda m: lambda t, output_size=None: m.conv(F.interpolate(t, size=(2 * t.shape[2],
                                                                                          2 * t.shape[3]))))(up)
        b = unet(x, torch.tensor([500]), ehs).sample
    assert torch.equal(a, b)


def _up_pairs():
    """every (in, out) pair of the nearest resizes the UNet makes at LATENTS, per side"""
    from mos_b200.engine import level_sizes
    pairs = set()
    for h, w in LATENTS:
        lv = level_sizes(h, w, 4)
        for (ho, wo), (hi, wi) in zip(lv[:-1], lv[1:]):
            pairs |= {(hi, ho), (wi, wo)}
    return sorted(pairs)


def _torch_nearest(n_in, n_out):
    """source index of each output position of F.interpolate(size=..., mode='nearest')"""
    src = torch.arange(n_in, dtype=torch.float32).view(1, 1, n_in, 1)
    return F.interpolate(src, size=(n_out, 1), mode='nearest').view(-1).long().tolist()


def test_nearest_index_rule_matches_torch():
    """The kernel's index rule (restated as norm_audit.nearest_src, which the launch audit's reference uses) equals
    F.interpolate(size=..., mode='nearest') for every resize of the test sizes and ~200 random (in, out) pairs, including
    ratios where the fp32 quotient rounds (odd in, non-power-of-two out)"""
    rng = random.Random(7)
    pairs = _up_pairs()
    assert (33, 65) in pairs and (9, 17) in pairs and (32, 63) in pairs and (1, 1) in pairs
    pairs += [(rng.randint(1, 300), 0) for _ in range(200)]
    pairs = [(i, o if o else rng.randint(1, 4 * i + 3)) for i, o in pairs]
    pairs += [(1000, 1999), (4095, 8191), (12345, 12346), (7, 3)]
    for n_in, n_out in pairs:
        got = [na.nearest_src(d, n_in, n_out) for d in range(n_out)]
        assert got == _torch_nearest(n_in, n_out), (n_in, n_out)


def test_nearest_rule_is_shift_at_exact_2x():
    for n in (1, 2, 3, 8, 33, 64, 1024):
        assert [na.nearest_src(d, n, 2 * n) for d in range(2 * n)] == [d >> 1 for d in range(2 * n)]


# ------------------------------------------------------------------------------------------- launch-audit references
def _rec(op, abi, x):
    return {'op': op, 'abi': abi, 'in': {'x': x}}


@pytest.mark.parametrize('H,W', [(65, 49), (33, 25), (17, 13), (9, 7), (1, 1), (8, 1), (63, 64)])
def test_im2col_reference_is_a_stride2_pad1_conv_at_odd_extents(H, W):
    """norm_audit's float64 im2col_s2 reference (pad 1), multiplied by a weight, is F.conv2d(stride=2, padding=1): the
    number of output pixels is ceil(H / 2) x ceil(W / 2) and every tap reads the right input pixel or a zero pad"""
    B, C, Co = 2, 8, 5
    g = torch.Generator().manual_seed(H * 100 + W)
    x = torch.randn(B, H, W, C, generator=g, dtype=torch.float64)
    wt = torch.randn(Co, C, 3, 3, generator=g, dtype=torch.float64)
    col = na.reference(_rec('mos_im2col_s2', dict(B=B, H=H, W=W, C=C, pad=1, ldx=C), x))['col'][0]
    Ho, Wo = (H + 1) // 2, (W + 1) // 2
    assert col.shape == (B, Ho, Wo, 9, C)
    got = torch.einsum('bhwtc,otc->bohw', col, wt.permute(0, 2, 3, 1).reshape(Co, 9, C))
    want = F.conv2d(x.permute(0, 3, 1, 2), wt, stride=2, padding=1)
    assert got.shape == want.shape
    assert torch.allclose(got, want, rtol=1e-12, atol=1e-12)


@pytest.mark.parametrize('H,W,Ho,Wo', [(9, 7, 17, 13), (33, 25, 65, 49), (32, 32, 63, 63), (1, 1, 1, 1), (4, 1, 8, 1),
                                       (8, 8, 16, 16)])
def test_upsample_reference_vs_interpolate(H, W, Ho, Wo):
    """norm_audit's reference of mos_upsample2x at an explicit output size is F.interpolate(size=..., mode='nearest')"""
    B, C = 2, 8
    x = torch.randn(B, H, W, C, generator=torch.Generator().manual_seed(H + W), dtype=torch.float64)
    y = na.reference(_rec('mos_upsample2x', dict(B=B, H=H, W=W, C=C, Ho=Ho, Wo=Wo, ldx=C), x))['y'][0]
    want = F.interpolate(x.permute(0, 3, 1, 2), size=(Ho, Wo), mode='nearest').permute(0, 2, 3, 1)
    assert torch.equal(y, want)


# ------------------------------------------------------------------------------------------------- refusals
REFUSED = [(520, 520), (1000, 1000), (904, 1808)]
ACCEPTED = [(576, 576), (640, 448), (768, 1536), (1024, 2048), (512, 512)]


@pytest.mark.parametrize('height,width', REFUSED + ACCEPTED)
def test_regional_size_rule(height, width):
    """check_region_sizes refuses exactly the sizes at which the region rule (reference :45-48) misreads a level"""
    from mixofshow.pipelines.pipeline_regionally_t2iadapter import check_region_sizes, region_feat_size
    from mos_b200.engine import level_sizes
    bad = any(region_feat_size(height, width, h * w) != (h, w) for h, w in level_sizes(height // 8, width // 8, 4))
    assert bad == ((height, width) in REFUSED)
    if bad:
        with pytest.raises(ValueError, match=f'{height} x {width}.*level'):
            check_region_sizes(height, width, 4)
    else:
        check_region_sizes(height, width, 4)


class _NoText:
    def __call__(self, *a, **k):
        raise AssertionError('text encoding ran before the size check')


@pytest.mark.parametrize('height,width', REFUSED)
def test_regional_pipeline_refuses_before_text_encoding(height, width):
    """the refusal comes at the call, before the tokenizer, text encoder or UNet are touched"""
    from types import SimpleNamespace
    from mixofshow.pipelines import pipeline_regionally_t2iadapter as pr
    unet = SimpleNamespace(config=SimpleNamespace(block_out_channels=(320, 640, 1280, 1280), in_channels=4),
                           down_blocks=torch.nn.ModuleList(), mid_block=torch.nn.Module(), up_blocks=torch.nn.ModuleList())
    pipe = pr.RegionallyT2IAdapterPipeline(unet=unet, tokenizer=_NoText(), text_encoder=_NoText())
    pipe.set_new_concept_cfg({})
    pipe._embed = _NoText()
    with pytest.raises(ValueError, match=f'{height} x {width}'):
        pipe(prompt=[['a photo', [('a cat', None, (0, 0, 1, 0.5))]]], height=height, width=width)


@pytest.mark.parametrize('h,w', [(65, 65), (64, 60), (4, 64)])
def test_train_engine_refuses_odd_latents_before_allocating(h, w):
    """TrainEngine's backward undoes exact halvings only; it refuses other latents before it touches the state dict or a
    device (the empty state dict and the CPU device would fail any later step)"""
    from mos_b200.train_engine import TrainEngine
    with pytest.raises(ValueError, match='multiples of 8'):
        TrainEngine({}, 2, h, w, lora={}, device='cpu')
