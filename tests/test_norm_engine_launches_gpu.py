"""Every norm / layout / elementwise launch of real engine walks, audited one by one (tests/norm_audit.py): implicit
pitches, a float64 reference with a derived per-element bound, per-unit rel-L2, the write window (pitch pads, the
GroupNorm workspace prefix), unchanged operands and a bit-identical second launch.

The walks are the eager walks of the other launch audits (tests/engine_walks.py): fp16 sampling at 64 x 64 (plain, and
a regional step with 3 boxes and emit_probs), at 96 x 192 with a whole-block LoRA, the drop-in RegionT2I_AttnProcessor,
bf16 training at the SD1.5 widths with the attention regulariser followed by the optimiser step, CLIP text encoding and
training, the VAE at 512 x 512 and the EDLoRAPipeline sampling loop (3 steps, CFG); and the product's own shapes: the
training step of bench.py train_leg at B = 2 (SD1.5 at 64 x 64, regulariser on all 16 cross layers without full_identity,
the 12-layer CLIP encoder trained in the same step, then AdamW and the LoRA re-pack over the three-group flat state) and
the validation pass (a 4-prompt CFG call, UNet batch 8, and the VAE decode of its 4 latents).  The last test prints one
row per path key and requires the keys reached to be exactly PATH_KEYS.
"""
import time

import pytest
import torch

import engine_walks as walks
import norm_audit as na

pytestmark = pytest.mark.gpu

# The path keys (norm_audit.norm_path) the walks reach on a 132-SM H100 (the GroupNorm cluster width k depends on the SM
# count through the 2 * SMs minimum grid), by engine call site:
#   engine.py:347 groupnorm (UNet, fp16 sampling / bf16 training): the cluster kernel at k = 1 / 2 / 4 / 8, vec 2 / 4;
#     vae_engine.py:161 at 512 x 512: the two-launch fallback with its partial workspace;
#   engine.py:355 / clip_train_engine.py:293 layernorm: C = 320 / 640 / 1280 and 768 (CLIP); the pipeline's CLIP
#     encoder runs 2 x 77 = 154 rows, a tail of the 8-row block;
#   train_engine.py:306 / 315 / 485 / 635 groupnorm_bwd (with SiLU, with add); :445 / :466 / :478 and
#     clip_train_engine.py:320 / 342 / 368 layernorm_bwd; :398 / clip_train_engine.py:245 lora_grad (R = 16, D / U
#     staged except the GEGLU projection); :586 masked_mse; :601 / :604 / :608 the attention regulariser;
#     dp.py:67 flat_adamw_step and :177 lora_pack (eng.optimizer_step);
#   engine.py:520-526 timestep_embedding and the time-MLP gemv (nb = 2); engine.py:584 / train_engine.py:504 /
#     vae_engine.py:226 / :273 conv_in; vae_engine.py:203 softmax_rows, :236 im2col pad 0, :255 vae_moments,
#     :270 conv1x1_nchw, :283 upsample2x;
#   pipeline_edlora.py:181 cfg_dpmpp_step with t_out and unet_in (the sampling loop);
#   engine.py:513 _region_rewrite and functional.py:162: region_combine in place over 3 regions;
#   train_engine.py: upsample2x, im2col pad 1, add_rows, geglu, upsample2x_bwd, col2im, conv_out_bwd, add_noise;
#   clip_engine.py / clip_train_engine.py: clip_embed, clip_embed_bwd, quick_gelu (in place), quick_gelu_fwd / _bwd.
# Only the product walks (train_sd15_full, validation_sd15) reach the keys marked "product": the regulariser without
# full_identity (train_engine.py:601, groups of 5 layers at 64^2 / 32^2 / 16^2 and the mid layer alone at 8^2), the
# time-MLP gemv at batch 8, GroupNorm at k = 2 (fp16, B = 8) and k = 8 / vec 4 (bf16 at 64 x 64), and lora_grad at
# R = 32 (CLIP, 32 x 77 rows) and R = 64 (UNet, 8192 rows).
PATH_KEYS = {
    'adamw',
    'add_noise',
    'add_rows|bf16',
    'attn_reg_grad',
    'attn_reg_group|L=1',                          # product
    'attn_reg_group|L=1|full',
    'attn_reg_group|L=3|full',
    'attn_reg_group|L=5',                          # product
    'attn_reg_total',
    'clip_embed',
    'cfg_step|cfg|t_out|unet_in',
    'clip_embed_bwd',
    'col2im',
    'conv1x1_nchw',
    'conv_in|bf16',
    'conv_in|fp16',
    'conv_out_bwd',
    'conv_out|bf16',
    'conv_out|fp16',
    'geglu_bwd',
    'geglu_fwd',
    'gemv|nb=2',
    'gemv|nb=2|act_out',
    'gemv|nb=8',                                   # product
    'gemv|nb=8|act_out',                           # product
    'gn_bwd|add',
    'gn_bwd|silu',
    'gn_bwd|silu|add',
    'gn|bf16|cluster|k=1|v4',
    'gn|bf16|cluster|k=1|v4|silu',
    'gn|bf16|cluster|k=4|v2|silu',
    'gn|bf16|cluster|k=4|v4',
    'gn|bf16|cluster|k=4|v4|silu',
    'gn|bf16|cluster|k=8|v2',
    'gn|bf16|cluster|k=8|v2|silu',
    'gn|bf16|cluster|k=8|v4',                      # product
    'gn|bf16|cluster|k=8|v4|silu',
    'gn|fp16|cluster|k=2|v2',                      # product
    'gn|fp16|cluster|k=2|v2|silu',                 # product
    'gn|fp16|cluster|k=2|v4',                      # product
    'gn|fp16|cluster|k=2|v4|silu',                 # product
    'gn|fp16|cluster|k=4|v4',
    'gn|fp16|cluster|k=4|v4|silu',
    'gn|fp16|cluster|k=8|v2',
    'gn|fp16|cluster|k=8|v2|silu',
    'gn|fp16|cluster|k=8|v4',
    'gn|fp16|cluster|k=8|v4|silu',
    'gn|fp16|fallback|silu',
    'im2col|pad=0',
    'im2col|pad=1',
    'ln_bwd|C=1280|add',
    'ln_bwd|C=320|add',
    'ln_bwd|C=640|add',
    'ln_bwd|C=768',
    'ln_bwd|C=768|add',
    'ln|bf16|C=1280',
    'ln|bf16|C=320',
    'ln|bf16|C=640',
    'ln|bf16|C=768',
    'ln|bf16|C=768|mtail',
    'ln|fp16|C=1280',
    'ln|fp16|C=320',
    'ln|fp16|C=640',
    'lora_grad|R=16|global',
    'lora_grad|R=16|staged',
    'lora_grad|R=32|staged',                       # product
    'lora_grad|R=64|staged',                       # product
    'lora_pack',
    'masked_mse',
    'quick_gelu',
    'quick_gelu_bwd',
    'quick_gelu_fwd',
    'region|fp16|n=3|inplace',
    'softmax_rows|fp16',
    'timestep_embedding',
    'upsample2x',
    'upsample2x_bwd',
    'vae_moments|fp16|noise',
}

STATS = na.Stats()
T0 = time.time()


def _audit():
    return na.Recorder(STATS)


@pytest.fixture(scope='module')
def sd15():
    return walks.sd15_pair()


def test_sample_64(cuda, sd15):
    walks.sample_64(sd15, _audit)


def test_sample_96x192_whole_block(cuda, sd15):
    walks.sample_96x192_whole_block(sd15, _audit)


def test_regional_step_with_probs(cuda, sd15):
    boxes = [(0.0, 0.0, 1.0, 0.4), (0.05, 0.35, 1.0, 0.7), (0.1, 0.65, 0.9, 1.0)]
    walks.sample_64(sd15, _audit, regions=boxes, emit_probs=True)


def test_functional_region_processor(cuda):
    """RegionT2I_AttnProcessor (functional.attention_block) on a 12 x 24 map: region_combine in place over its output"""
    from mixofshow.pipelines.pipeline_regionally_t2iadapter import RegionT2I_AttnProcessor
    from oracle.unet import Attention
    torch.manual_seed(6)
    attn_x = Attention(320, 768, heads=8, dim_head=40).cuda()
    g = torch.Generator().manual_seed(7)
    hs = torch.randn(2, 288, 320, generator=g).cuda()
    ehs = torch.randn(2, 77, 768, generator=g).cuda()
    boxes = [(0.0, 0.0, 1.0, 0.4), (0.05, 0.35, 1.0, 0.7), (0.1, 0.65, 0.9, 1.0)]
    rl = [(torch.randn(2, 77, 768, generator=g).cuda(), b) for b in boxes]
    with _audit():
        RegionT2I_AttnProcessor(0)(attn_x, hs, encoder_hidden_states=ehs, region_list=rl, height=96, width=192)
        torch.cuda.synchronize()


def test_train_with_attention_regulariser_and_optimizer_step(cuda):
    walks.train_sd15_channels_whole_block(_audit, attn_reg_weight=0.05, optimizer_step=True)


def test_vae_512(cuda):
    walks.vae_512(_audit)


def test_sampling_loop(cuda, tmp_path):
    walks.sampling_loop(_audit, tmp_path)


def test_clip_text_and_train(cuda):
    walks.clip_text_and_train(_audit, cuda)


def test_train_sd15_full(cuda):
    walks.train_sd15_full(_audit)


def test_validation_sd15(cuda):
    walks.validation_sd15(_audit)


def test_coverage_table(cuda):
    print(f'\nnorm / elementwise launch audit ({time.time() - T0:.0f} s, '
          f'{torch.cuda.get_device_properties(0).multi_processor_count} SMs)\n' + STATS.table())
    assert not STATS.failures, '\n'.join(STATS.failures[:30])
    reached = set(STATS.rows)
    assert reached == PATH_KEYS, (f'reached but not listed: {sorted(reached - PATH_KEYS)}; '
                                  f'listed but not reached: {sorted(PATH_KEYS - reached)}')
