"""Every attention-family launch of real engine walks, audited one by one (tests/attention_audit.py): the zero pads and
transposed copies the kernel reads, a float64 reference with a derived per-element bound, per-tile rel-L2, the write
window, unchanged operands and a bit-identical second launch.

The end-to-end tests compare one global rel-L2 or LoRA gradients at 8e-2: one wrong (batch, head, 128-query) tile out of
512, a wrong dK of one head or a stale transposed copy pass them.  The walks are eager (use_graph=False):
- fp16 sampling at 64 x 64: SD1.5 UNet, CFG batch 2, fused attention LoRA;
- fp16 sampling at 96 x 192 with a whole-block LoRA: 18432 / 4608 / 1152 / 288 tokens;
- a regional step (UNetEngine.set_regions, 3 boxes, emit_probs=True): per-region cross-attention and `probs`; and the
  drop-in RegionT2I_AttnProcessor (mos_b200/functional.py) on a 12 x 24 feature map with 3 regions;
- bf16 training at the SD1.5 widths, 16 x 16, B = 2, with the attention regulariser (pcols, pos, gcols);
- CLIP: CLIPTextEngine (causal forward), CLIPTrainEngine forward + backward (causal lse2, causal backward, dq | dk | dv
  thirds of one storage);
- the product's training step (bench.py train_leg at B = 2): bf16 SD1.5 at 64 x 64 (4096 / 1024 / 256 / 64 tokens) with
  the regulariser on all 16 cross layers and the 12-layer CLIP encoder over 32 sequences;
- the product's validation pass: a 4-prompt CFG call (UNet batch 8: B H = 64) and the VAE decode of its 4 latents.
The last test prints one row per path key and requires the keys reached to be exactly PATH_KEYS.
"""
import time

import pytest
import torch

import attention_audit as aa
import engine_walks as walks

pytestmark = pytest.mark.gpu

# The path keys (attention_audit.attn_path) the walks reach, by engine call site:
#   engine.py UNetEngine.transformer (attn1, attn2 with probs when emit_probs) and _region_rewrite: fwd|fp16 at
#     4096 / 1024 / 256 / 64 tokens (64 x 64) and 18432 / 4608 / 1152 / 288 (96 x 192); 77 text keys are one tile for
#     d = 40 / 160 and the multi-tile kernel for d = 80;
#   functional.py attention_block (RegionT2I_AttnProcessor, 288 tokens, d = 40): the fp16 d = 40 keys with a query tail;
#   train_engine.py transformer_train (attention_train, pcols on attn2), _attn_bwd (heads_transpose, attn_delta,
#     attention_bwd with gcols on attn2), _cross_kv_train (heads_transpose of the 77-token text K / V):
#     fwd|bf16 / bwd|bf16 / delta / transpose at 256 / 64 / 16 / 4 tokens;
#   clip_engine.py forward and clip_train_engine.py forward_train (attention_causal, without and with lse2), backward
#     (heads_transpose, attn_delta, causal attention_bwd into the dqkv thirds): the D=80 causal keys.
# Only the product walks (train_sd15_full, validation_sd15) reach the keys marked "product": the toy training walk has
# d = 80 / 160 only at 64 / 16 / 4 tokens (query tails), the 64 x 64 step at 1024 (d = 80) and 256 / 64 (d = 160) tokens,
# so the d = 80 / 160 self-attention forward and backward run tail-free multi-tile launches, the cross-attention full
# query tiles, and the 64-token d = 160 backward a one-tile launch with a query tail but no key tail.
PATH_KEYS = {
    # UNetEngine, fp16
    'fwd|fp16|D=40|multi',
    'fwd|fp16|D=40|one|ktail',
    'fwd|fp16|D=40|one|probs|ktail',
    'fwd|fp16|D=80|multi',
    'fwd|fp16|D=80|multi|ktail',
    'fwd|fp16|D=80|multi|probs|ktail',
    'fwd|fp16|D=160|multi',
    'fwd|fp16|D=160|multi|qtail|ktail',
    'fwd|fp16|D=160|one|ktail',
    'fwd|fp16|D=160|one|probs|ktail',
    'fwd|fp16|D=160|one|probs|qtail|ktail',
    'fwd|fp16|D=160|one|qtail|ktail',
    # functional.attention_block
    'fwd|fp16|D=40|multi|qtail|ktail',
    'fwd|fp16|D=40|one|qtail|ktail',
    # TrainEngine, bf16
    'fwd|bf16|D=40|multi|lse2',
    'fwd|bf16|D=40|one|lse2|pcols|ktail',
    'fwd|bf16|D=80|multi|lse2',                     # product
    'fwd|bf16|D=80|multi|lse2|pcols|ktail',         # product
    'fwd|bf16|D=80|multi|lse2|qtail|ktail',
    'fwd|bf16|D=80|multi|lse2|pcols|qtail|ktail',
    'fwd|bf16|D=160|one|lse2|qtail|ktail',
    'fwd|bf16|D=160|multi|lse2',                    # product
    'fwd|bf16|D=160|one|lse2|pcols|ktail',          # product
    'fwd|bf16|D=160|one|lse2|pcols|qtail|ktail',
    'bwd|bf16|D=40|multi',
    'bwd|bf16|D=40|multi|gcols|ktail',
    'bwd|bf16|D=80|one|qtail',
    'bwd|bf16|D=80|multi',                          # product
    'bwd|bf16|D=80|multi|gcols|ktail',              # product
    'bwd|bf16|D=80|multi|gcols|qtail|ktail',
    'bwd|bf16|D=160|one|qtail|ktail',
    'bwd|bf16|D=160|one|qtail',                     # product
    'bwd|bf16|D=160|multi',                         # product
    'bwd|bf16|D=160|multi|gcols|ktail',             # product
    'bwd|bf16|D=160|multi|gcols|qtail|ktail',
    'delta|D=40',
    'delta|D=40|pcols',
    'delta|D=80',
    'delta|D=80|pcols',
    'delta|D=160',
    'delta|D=160|pcols',
    'transpose|DP=64|DV=48',
    'transpose|DP=64|DV=48|rtail',
    'transpose|DP=128|DV=80',
    'transpose|DP=128|DV=80|rtail',
    'transpose|DP=192|DV=160',
    'transpose|DP=192|DV=160|rtail',
    # CLIPTextEngine / CLIPTrainEngine
    'fwd|bf16|D=80|one|causal|qtail|ktail',
    'fwd|bf16|D=80|one|causal|lse2|qtail|ktail',
    'bwd|bf16|D=80|multi|causal|qtail|ktail',
}

STATS = aa.Stats()
T0 = time.time()


def _audit():
    return aa.Recorder(STATS)


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
    """RegionT2I_AttnProcessor (functional.attention_block) on a 12 x 24 map (288 tokens, d = 40), self and 3 regions"""
    from mixofshow.pipelines.pipeline_regionally_t2iadapter import RegionT2I_AttnProcessor
    from oracle.unet import Attention
    torch.manual_seed(6)
    attn_s = Attention(320, None, heads=8, dim_head=40).cuda()
    attn_x = Attention(320, 768, heads=8, dim_head=40).cuda()
    g = torch.Generator().manual_seed(7)
    hs = torch.randn(2, 288, 320, generator=g).cuda()
    ehs = torch.randn(2, 77, 768, generator=g).cuda()
    boxes = [(0.0, 0.0, 1.0, 0.4), (0.05, 0.35, 1.0, 0.7), (0.1, 0.65, 0.9, 1.0)]
    rl = [(torch.randn(2, 77, 768, generator=g).cuda(), b) for b in boxes]
    with _audit():
        RegionT2I_AttnProcessor(0)(attn_s, hs, encoder_hidden_states=None, region_list=[], height=96, width=192)
        RegionT2I_AttnProcessor(0)(attn_x, hs, encoder_hidden_states=ehs, region_list=rl, height=96, width=192)
        torch.cuda.synchronize()


def test_train_with_attention_regulariser(cuda):
    walks.train_sd15_channels_whole_block(_audit, attn_reg_weight=0.05)


def test_clip_text_and_train(cuda):
    walks.clip_text_and_train(_audit, cuda)


def test_train_sd15_full(cuda):
    walks.train_sd15_full(_audit)


def test_validation_sd15(cuda):
    walks.validation_sd15(_audit)


def test_coverage_table(cuda):
    print(f'\nattention launch audit ({time.time() - T0:.0f} s)\n' + STATS.table())
    assert not STATS.failures, '\n'.join(STATS.failures[:30])
    reached = set(STATS.rows)
    assert reached == PATH_KEYS, (f'reached but not listed: {sorted(reached - PATH_KEYS)}; '
                                  f'listed but not reached: {sorted(PATH_KEYS - reached)}')
