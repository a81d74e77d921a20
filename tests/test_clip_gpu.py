"""CLIP text encoder on the GPU (SURVEY.md 8f rank 1) vs the library the reference itself calls: transformers
`CLIPTextModel` (random-init from `CLIPTextConfig` with the SD1.5 sizes; fp32 on CPU).  Tolerances: bf16 weights and
activations through 12 pre-LN layers: rel-L2 <= 2e-2 on the final hidden state (the UNet path measures 8e-3 .. 1e-2)."""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu


def rel_l2(a, b):
    a, b = a.float().cpu(), b.float().cpu()
    return ((a - b).norm() / b.norm().clamp_min(1e-12)).item()


@pytest.mark.parametrize('n_seq,n', [(3, 77), (16, 77), (2, 40), (1, 128)])
def test_attention_causal_padded_heads(cuda, n_seq, n):
    """12 heads of 64 dims run as head_dim 80 with zero padding and scale 64^-0.5; row q only sees keys <= q."""
    from mos_b200 import ops
    H, d, dh = 12, 64, 80
    g = torch.Generator().manual_seed(0)
    q, k, v = (torch.randn(n_seq, H, n, d, generator=g).to(torch.bfloat16).to(cuda) for _ in range(3))
    n8 = (n + 7) // 8 * 8
    Q = torch.zeros(n_seq * H, n, 128, device=cuda, dtype=torch.bfloat16)
    K = torch.zeros(n_seq * H, n, 128, device=cuda, dtype=torch.bfloat16)
    Vt = torch.zeros(n_seq * H, dh, n8, device=cuda, dtype=torch.bfloat16)
    Q[..., :d] = q.reshape(n_seq * H, n, d)
    K[..., :d] = k.reshape(n_seq * H, n, d)
    Vt[:, :d, :n] = v.reshape(n_seq * H, n, d).transpose(1, 2)
    out = torch.full((n_seq, n, H * dh), float('nan'), device=cuda, dtype=torch.bfloat16)
    ops.attention_causal(Q, K, Vt, out, batch=n_seq, heads=H, head_dim=dh, n=n, scale=d ** -0.5)
    torch.cuda.synchronize()
    ref = F.scaled_dot_product_attention(q.float(), k.float(), v.float(), is_causal=True)   # [n_seq, H, n, d]
    got = out.view(n_seq, n, H, dh)
    assert got[..., d:].abs().max().item() == 0.0            # pad columns of every head stay zero
    assert rel_l2(got[..., :d].permute(0, 2, 1, 3), ref) < 8e-3


def test_quick_gelu_and_embed(cuda):
    from mos_b200 import ops
    g = torch.Generator().manual_seed(1)
    x = (torch.randn(100, 3200, generator=g) * 2).to(torch.bfloat16).to(cuda)
    ref = x.float() * torch.sigmoid(1.702 * x.float())
    ops.quick_gelu(x, M=100, C=3200)
    assert rel_l2(x, ref) < 3e-3
    tok = torch.randn(500, 768, generator=g).to(cuda)
    pos = torch.randn(77, 768, generator=g).to(cuda)
    ids = torch.randint(0, 500, (3 * 77,), generator=g).to(torch.int32).to(cuda)
    out = torch.full((3 * 77, 800), float('nan'), device=cuda, dtype=torch.bfloat16)
    ops.clip_embed(ids, tok, pos, out, T=77, C=768)
    ref = tok[ids.long()] + pos.repeat(3, 1)
    assert rel_l2(out[:, :768], ref) < 3e-3 and out[:, 768:].abs().max().item() == 0.0


def _clip(layers):
    from transformers import CLIPTextConfig, CLIPTextModel
    cfg = CLIPTextConfig(vocab_size=49408, hidden_size=768, intermediate_size=3072, num_hidden_layers=layers,
                         num_attention_heads=12, max_position_embeddings=77)
    torch.manual_seed(0)
    return CLIPTextModel(cfg).eval()


@pytest.mark.parametrize('layers,with_lora,merged', [(2, False, False), (2, True, False), (2, True, True),
                                                     (12, True, False)])
def test_clip_text_engine_vs_transformers(cuda, layers, with_lora, merged):
    from mos_b200.clip_engine import CLIPTextEngine
    from oracle import inject
    model = _clip(layers)
    sd = {k: v.clone() for k, v in model.state_dict().items()}
    lora = inject.random_lora_state(model, seed=7, where='CLIPAttention', up_std=0.05) if with_lora else None
    n_seq = 16
    g = torch.Generator().manual_seed(3)
    ids = torch.randint(0, 49407, (n_seq, 77), generator=g)
    ids[:, 0] = 49406
    ids[:, 9:] = 49407                                     # BOS, 8 prompt tokens, EOS padding (as the tokenizer pads)
    if with_lora:
        inject.inject_lora(model, lora, 0.8)               # y = orig(x) + alpha * up(down(x)), edlora.py:244-246
    with torch.no_grad():
        ref = model(ids)[0]                                # last_hidden_state, fp32 CPU
    eng = CLIPTextEngine(sd, n_seq, lora=lora, lora_alpha=0.8, merge_lora=merged)
    out = eng(ids)
    torch.cuda.synchronize()
    e = rel_l2(out, ref)
    print(f'CLIP text encoder, {layers} layers, lora={with_lora} merged={merged}: rel-L2 {e:.3e}, {eng.launches} launches')
    assert torch.isfinite(out).all()
    assert e < 2e-2
    # the un-merged LoRA must matter (the test would otherwise pass with the LoRA path broken)
    if with_lora and not merged:
        base = CLIPTextEngine(sd, n_seq)(ids)
        assert rel_l2(base, ref) > 2 * e


@pytest.mark.gpu
def test_clip_container_unpadded_ids(cuda):
    """gradient_fusion.py:190-199 calls the text encoder with UN-padded prompts, one at a time: the container pads to the
    engine's fixed length (the encoder is causal) and returns the first L positions - equal to transformers on the same
    ids, and to the prefix of the padded call."""
    from mixofshow.models.clip_b200 import CLIPTextModel as GpuClip
    model = _clip(2)
    enc = GpuClip({k: v.clone() for k, v in model.state_dict().items()})
    ids = torch.tensor([[49406, 320, 1125, 539, 320, 49408 % 49407, 49407]])      # BOS, 5 words, EOS: L = 7
    with torch.no_grad():
        ref = model(ids)[0]
    out = enc(ids.cuda())[0]
    assert tuple(out.shape) == (1, 7, 768)
    assert rel_l2(out, ref) < 2e-2
    padded = torch.cat([ids, ids[:, -1:].expand(1, 70)], 1)
    full = enc(padded.cuda())[0]
    assert torch.equal(full[:, :7], out)
