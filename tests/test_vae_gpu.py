"""VAE encoder / decoder on the GPU (`mos_b200/vae_engine.py`, SURVEY.md 8f rank 2) against the fp32 oracle restatement of
diffusers' AutoencoderKL (oracle/vae.py; "parity unpinned": diffusers is absent and the reference has no vectors for this
boundary).  Reference call sites: `vae.encode(images).latent_dist.sample() * 0.18215` (trainer_edlora.py:203-204) and
`vae.decode(latents / 0.18215).sample` (pipeline_edlora.py:303-313).

Tolerances: fp16 operands, fp32 accumulation / statistics / softmax: rel-L2 <= 5e-3 on the posterior mean, the sampled
latents and the decoded image (the UNet path measures ~1e-3 at comparable depth)."""
import pytest
import torch

pytestmark = pytest.mark.gpu


def rel_l2(a, b):
    a, b = a.float().cpu(), b.float().cpu()
    return ((a - b).norm() / b.norm().clamp_min(1e-12)).item()


def _check_encode_decode(cuda, cfg_name, B, H, W, decode=True):
    from gpu_helpers import gn_path, rup
    from mos_b200.vae_engine import VAEEngine
    from oracle import vae as ov
    cfg = ov.TINY_VAE if cfg_name == 'tiny' else None
    ref = ov.build_vae(0, cfg)
    full = dict(ov.SD15_VAE, **(cfg or {}))
    sd = {k: v.detach().clone() for k, v in ref.state_dict().items()}
    c0 = full['block_out_channels'][0]
    if H * W >= 512 * 512:
        assert gn_path(B, H * W, c0, rup(c0, 160), c0) == 'fallback'
        ref = ref.to(cuda)
    dev = next(ref.parameters()).device
    eng = VAEEngine(sd, B, H, W, block_out=full['block_out_channels'], layers=full['layers_per_block'])
    g = torch.Generator().manual_seed(1)
    img = torch.rand(B, 3, H, W, generator=g) * 2 - 1
    d = 2 ** (len(full['block_out_channels']) - 1)
    noise = torch.randn(B, 4, H // d, W // d, generator=g)
    with torch.no_grad():
        mean_ref, logvar_ref = ref.moments(img.to(dev))
        lat_ref = ref.encode_sample(img.to(dev), noise.to(dev)) * 0.18215
    mean, logvar, lat = eng.encode(img.cuda(), noise=noise.cuda())
    torch.cuda.synchronize()
    e_m, e_v, e_l = rel_l2(mean, mean_ref), rel_l2(logvar, logvar_ref), rel_l2(lat, lat_ref)
    n_enc = eng.launches
    msg = f'VAE [{cfg_name}] {B}x3x{H}x{W}: mean rel-L2 {e_m:.3e}, logvar {e_v:.3e}, latents {e_l:.3e} ({n_enc} launches)'
    e_d = 0.0
    if decode:
        z = torch.randn(B, 4, H // d, W // d, generator=g)
        with torch.no_grad():
            dec_ref = ref.decode(z.to(dev))
        dec = eng.decode(z.cuda())
        torch.cuda.synchronize()
        e_d = rel_l2(dec, dec_ref)
        msg += f'; decode rel-L2 {e_d:.3e} ({eng.launches} launches)'
    print(msg)
    assert max(e_m, e_v, e_l, e_d) < 5e-3


@pytest.mark.parametrize('cfg_name,B,H,W', [('tiny', 2, 64, 64), ('tiny', 1, 64, 128), ('sd15', 1, 256, 256)])
def test_vae_encode_decode(cuda, cfg_name, B, H, W):
    _check_encode_decode(cuda, cfg_name, B, H, W)


# 512 x 512 is the resolution training encodes (B = 2 per GPU, encode only) and the pipeline decodes; it is the only size
# at which the VAE's full-resolution GroupNorms take the two-launch fallback.  Its fp32 oracle runs on the GPU (TF32 off).
@pytest.mark.parametrize('B,decode', [(1, True), (2, False)], ids=['B1', 'B2-encode'])
def test_vae_encode_decode_512(cuda, B, decode):
    _check_encode_decode(cuda, 'sd15', B, 512, 512, decode)


def test_vae_container_call_shapes(cuda, tmp_path):
    """`AutoencoderKL.from_pretrained(path, subfolder='vae')`, `.encode(x).latent_dist.sample()`, `.decode(z).sample` and the
    old attention key names (query / key / value / proj_attn) of pre-0.18 checkpoints."""
    from mixofshow.models.vae_b200 import AutoencoderKL
    from mixofshow.utils import model_io
    from oracle import vae as ov
    ref = ov.build_vae(0, ov.TINY_VAE)
    old = {}
    ren = {'to_q': 'query', 'to_k': 'key', 'to_v': 'value', 'to_out.0': 'proj_attn'}
    for k, v in ref.state_dict().items():
        for new_n, old_n in ren.items():
            if f'.attentions.0.{new_n}.' in k:
                k = k.replace(f'.attentions.0.{new_n}.', f'.attentions.0.{old_n}.')
        old[k] = v.detach()
    vae = AutoencoderKL(old, block_out_channels=ov.TINY_VAE['block_out_channels'], layers_per_block=1)
    model_io.save_vae(vae, str(tmp_path))
    vae2 = AutoencoderKL.from_pretrained(str(tmp_path), subfolder='vae')
    img = torch.rand(1, 3, 64, 64, generator=torch.Generator().manual_seed(2)) * 2 - 1
    dist = vae2.encode(img.cuda()).latent_dist
    with torch.no_grad():
        mean_ref, _ = ref.moments(img)
    assert rel_l2(dist.mode(), mean_ref) < 5e-3
    s = dist.sample(generator=torch.Generator().manual_seed(0))
    assert tuple(s.shape) == (1, 4, 32, 32) and torch.isfinite(s).all()
    out = vae2.decode(s / 0.18215 * 0.18215).sample
    assert tuple(out.shape) == (1, 3, 64, 64)


def test_pipeline_decodes_to_pil(cuda):
    """EDLoRAPipeline.__call__ with output_type='pil' (the reference default, pipeline_edlora.py:303-313): latents / 0.18215
    -> GPU VAE decode -> [0,1] clamp -> PIL, so that `.images[0].save(...)` works as in the reference's scripts."""
    from mixofshow.models.unet_b200 import UNet2DConditionModel
    from mixofshow.models.vae_b200 import AutoencoderKL
    from mixofshow.pipelines.pipeline_edlora import EDLoRAPipeline
    from oracle import unet as ou
    from oracle import vae as ov
    ref = ou.build_unet(0, ou.TINY)
    unet = UNet2DConditionModel(block_out_channels=ou.TINY['block_out_channels'], layers_per_block=ou.TINY['layers_per_block'])
    unet.load_state_dict(ref.state_dict())
    vref = ov.build_vae(0, ov.TINY_VAE)
    vae = AutoencoderKL({k: v.detach() for k, v in vref.state_dict().items()},
                        block_out_channels=ov.TINY_VAE['block_out_channels'], layers_per_block=1)
    pipe = EDLoRAPipeline(vae=vae, unet=unet).to('cuda')
    pipe.set_new_concept_cfg({})
    g = torch.Generator().manual_seed(3)
    lat = torch.randn(1, 4, 16, 16, generator=g)
    pe, ne = torch.randn(1, 16, 77, 768, generator=g), torch.randn(1, 77, 768, generator=g)
    kw = dict(prompt_embeds=pe.cuda(), negative_prompt_embeds=ne.cuda(), height=32, width=32, num_inference_steps=3,      # vae_scale_factor = 2 for the tiny VAE
              guidance_scale=3.0)
    lat_out = pipe(latents=lat.clone(), output_type='latent', **kw).images
    imgs = pipe(latents=lat.clone(), output_type='pil', **kw).images
    assert isinstance(imgs, list) and imgs[0].size == (32, 32)            # TINY_VAE upsamples x2
    with torch.no_grad():
        dec = vref.decode(lat_out.cpu() / 0.18215)
    want = ((dec / 2 + 0.5).clamp(0, 1)[0].permute(1, 2, 0) * 255).round()
    import numpy as np
    got = torch.from_numpy(np.asarray(imgs[0]).astype('float32'))
    assert (got - want).abs().max().item() <= 2.0                         # 8-bit levels
