"""Every GEMM launch of real engine walks, audited one by one (tests/gemm_audit.py): float64 reference, per-element bound,
per-tile rel-L2, write window, unchanged operands and a bit-identical second launch.

The end-to-end tests cannot see one bad launch: a wrong tile out of 512, a wrong batch bias on a tail patch or a stray
write into a Q/K pad column all vanish inside their eps / gradient bounds.  The walks are eager (use_graph=False):
- fp16 sampling at 64 x 64: SD1.5 UNet, CFG batch 2, fused attention LoRA, with the per-prompt text K/V update;
- fp16 sampling at 96 x 192 (conv height / batch tails) with a fused whole-block LoRA (`where: Transformer2DModel`);
- bf16 training: TrainEngine.forward_backward at the SD1.5 channels, one layer per block, 16 x 16, B = 2, whole-block LoRA;
- CLIP: CLIPTextEngine, 12 layers, fused CLIPAttention LoRA; CLIPTrainEngine forward + backward, CLIPEncoderLayer LoRA;
- VAE encode + decode at 512 x 512, B = 1;
- gradient fusion: Gram recording of one spatial stage with whole-block keys;
- the product's training step (bench.py train_leg at B = 2): SD1.5 UNet at 64 x 64 with an Attention LoRA, the regulariser
  on all 16 cross layers, the 12-layer CLIP encoder trained in the same step (d(text embeddings) GEMMs, CLIP backward from
  the UNet's pitched d_ehs), then the optimiser step;
- the product's validation pass: a 4-prompt CFG call (UNet batch 8, 2 steps) and the VAE decode of its 4 latents at 512;
- the opt-in paths: a child process repeats the 64 x 64 walk with MOS_SPLITK_FUSED=1 MOS_L2_PREFETCH=1 (both read at
  import); its launches are audited too, and its eps must be bit-identical to the default walk's (the in-kernel finalize
  sums the partials in the same order as mos_splitk_finalize).
The last test prints one row per path key and requires the keys reached to be exactly PATH_KEYS.
"""
import json
import os
import subprocess
import sys
import time

import pytest
import torch

if __name__ == '__main__':
    _root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    sys.path[:0] = [_root, os.path.join(_root, 'mix-of-show_b200'), os.path.dirname(os.path.abspath(__file__))]

import engine_walks as walks  # noqa: E402
import gemm_audit as ga  # noqa: E402

pytestmark = pytest.mark.gpu

# The path keys (gemm_audit.gemm_path) the walks reach, each checked against its engine call site: f32+acc is the Gram
# accumulation (gradient_fusion.py GramRecorder), f32 the VAE attention scores (vae_engine.py S = Q K^T); geglu is ff1
# (engine.py, LoRA with the whole-block placement); heads / heads_vt are the q | k | v, q and text k | v projections of the
# UNet, VAE, CLIP and training engines and the training engine's attention-output backward (copy-out where the token count
# is neither 64 nor a multiple of 128: 77 text tokens, the 288-token 12 x 24 level of a 96 x 192 latent, and 16 / 4 at
# the 4 x 4 / 2 x 2 levels of a 16 x 16 training latent); partial and splitk_finalize are the split-K launches of
# UNetEngine.gemm (fused: MOS_SPLITK_FUSED=1); rows / rows+res_smem are every other linear and conv.  No engine launch
# reaches the global-memory residual or copied-out row output.
# Only the product walks (train_sd15_full, validation_sd15) reach the keys marked "product": at 64 x 64 (M = 8192) the
# training convs have enough tiles to skip split-K (UNetEngine._splits), so conv1 stores directly with the time-embedding
# batch bias (train_engine.py:290), conv2 with the staged residual (:293), and so do the backward convs (:303 / :308 /
# :658; :303 and :658 read dOut at a pitched lda); the attn1 q | k | v projections write 4096 / 1024 tokens through the bf16 head-split TMA path.
PATH_KEYS = {
    'f32+acc|global|fp16',
    'f32|global|fp16',
    'geglu|tma|fp16',
    'geglu|tma|fp16|lora',
    'heads_vt|copy|bf16|lora|T=77',
    'heads_vt|copy|fp16|T=77',
    'heads_vt|copy|fp16|lora|T=288',
    'heads_vt|copy|fp16|lora|T=77',
    'heads_vt|tma|fp16|T=256',
    'heads_vt|tma|fp16|T=4096',
    'heads_vt|tma|fp16|T=64',
    'heads_vt|tma|fp16|lora|T=1024',
    'heads_vt|tma|fp16|lora|T=1152',
    'heads_vt|tma|fp16|lora|T=18432',
    'heads_vt|tma|fp16|lora|T=256',
    'heads_vt|tma|fp16|lora|T=4096',
    'heads_vt|tma|fp16|lora|T=4608',
    'heads_vt|tma|fp16|lora|T=64',
    'heads|copy|bf16|lora|T=16',
    'heads|copy|bf16|lora|T=4',
    'heads|copy|bf16|lora|T=77',
    'heads|copy|fp16|lora|T=288',
    'heads|tma|bf16|lora|T=1024',                  # product
    'heads|tma|bf16|lora|T=256',
    'heads|tma|bf16|lora|T=4096',                  # product
    'heads|tma|bf16|lora|T=64',
    'heads|tma|fp16|T=256',
    'heads|tma|fp16|T=64',
    'heads|tma|fp16|lora|T=1024',
    'heads|tma|fp16|lora|T=1152',
    'heads|tma|fp16|lora|T=18432',
    'heads|tma|fp16|lora|T=256',
    'heads|tma|fp16|lora|T=4096',
    'heads|tma|fp16|lora|T=4608',
    'heads|tma|fp16|lora|T=64',
    'partial|global|bf16',
    'partial|global|bf16|conv',
    'partial|global|fp16',
    'partial|global|fp16|conv',
    'partial|global|fp16|conv|fused',
    'partial|global|fp16|fused',
    'rows+res_smem|tma|bf16',
    'rows+res_smem|tma|bf16|conv',                 # product
    'rows+res_smem|tma|bf16|lora',
    'rows+res_smem|tma|fp16',
    'rows+res_smem|tma|fp16|conv',
    'rows+res_smem|tma|fp16|lora',
    'rows|tma|bf16',
    'rows|tma|bf16|conv',                          # product
    'rows|tma|bf16|conv|bb',                       # product
    'rows|tma|bf16|lora',
    'rows|tma|fp16',
    'rows|tma|fp16|conv',
    'rows|tma|fp16|conv|bb',
    'rows|tma|fp16|lora',
    'splitk_finalize|bf16',
    'splitk_finalize|bf16|bb',
    'splitk_finalize|bf16|res',
    'splitk_finalize|fp16',
    'splitk_finalize|fp16|bb',
    'splitk_finalize|fp16|res',
}

STATS = ga.Stats()
EPS = {}
T0 = time.time()


def _audited(fn):
    with ga.Recorder(STATS):
        out = fn()
        torch.cuda.synchronize()
    return out


@pytest.fixture(scope='module')
def sd15():
    return walks.sd15_pair()


def walk_sample64(sd15_pair, stats):
    return walks.sample_64(sd15_pair, lambda: ga.Recorder(stats))


def test_sample_64(cuda, sd15):
    EPS['default'] = walk_sample64(sd15, STATS)


def test_sample_96x192_whole_block(cuda, sd15):
    walks.sample_96x192_whole_block(sd15, lambda: ga.Recorder(STATS))


def test_train_sd15_channels_whole_block(cuda):
    walks.train_sd15_channels_whole_block(lambda: ga.Recorder(STATS))


def test_clip_text_and_train(cuda):
    walks.clip_text_and_train(lambda: ga.Recorder(STATS), cuda)


def test_vae_512(cuda):
    walks.vae_512(lambda: ga.Recorder(STATS))


def test_fusion_gram_whole_block(cuda):
    from gradient_fusion import GramRecorder
    from mos_b200.engine import UNetEngine, ehs_to_layer_major
    from oracle import inject
    from oracle import unet as ou
    unet = ou.build_unet(0, ou.TINY)
    sd = {k: v.clone() for k, v in unet.state_dict().items()}
    lora = inject.random_lora_state(unet, seed=10, where='Transformer2DModel', up_std=0.05)
    H = 16
    g = torch.Generator().manual_seed(3)
    lat = torch.randn(1, 4, H, H, generator=g)
    ehs = torch.randn(1, 4, 77, 768, generator=g)
    eng = UNetEngine(sd, 1, H, H, lora=lora, lora_alpha=0.8, merge_lora=True, use_graph=False,
                     block_out=ou.TINY['block_out_channels'], layers=1)
    eng.gram_rec = GramRecorder(cuda)
    _audited(lambda: eng.forward(lat.cuda(), torch.tensor([501.0]).cuda(), ehs_to_layer_major(ehs.cuda(), 4)))


def test_opt_in_paths_child(cuda, tmp_path):
    """MOS_SPLITK_FUSED=1 MOS_L2_PREFETCH=1: the same 64 x 64 walk in a child process, audited there"""
    env = dict(os.environ, MOS_SPLITK_FUSED='1', MOS_L2_PREFETCH='1')
    r = subprocess.run([sys.executable, os.path.abspath(__file__), str(tmp_path)], env=env, capture_output=True,
                       text=True)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-4000:]
    with open(tmp_path / 'stats.json') as f:
        STATS.merge(json.load(f))
    eps = torch.load(tmp_path / 'eps.pt')
    assert 'default' in EPS
    assert torch.equal(eps.view(torch.int32), EPS['default'].cpu().view(torch.int32)), \
        'the in-kernel split-K finalize changed eps'


def test_train_sd15_full(cuda):
    walks.train_sd15_full(lambda: ga.Recorder(STATS))


def test_validation_sd15(cuda):
    walks.validation_sd15(lambda: ga.Recorder(STATS))


def test_coverage_table(cuda):
    print(f'\nGEMM launch audit ({time.time() - T0:.0f} s)\n' + STATS.table())
    assert not STATS.failures, '\n'.join(STATS.failures[:30])
    reached = set(STATS.rows)
    assert reached == PATH_KEYS, (f'reached but not listed: {sorted(reached - PATH_KEYS)}; '
                                  f'listed but not reached: {sorted(PATH_KEYS - reached)}')


if __name__ == '__main__':
    torch.backends.cuda.matmul.allow_tf32 = False
    _stats = ga.Stats()
    _eps = walk_sample64(walks.sd15_pair(), _stats)
    torch.save(_eps.cpu(), os.path.join(sys.argv[1], 'eps.pt'))
    with open(os.path.join(sys.argv[1], 'stats.json'), 'w') as f:
        json.dump({'rows': _stats.rows, 'failures': _stats.failures}, f)
