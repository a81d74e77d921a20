"""Text-encoder half of the ED-LoRA training step on the GPU (`mos_b200/clip_train_engine.py`) against fp32 autograd through
the library the reference itself calls (transformers `CLIPTextModel`, random-init at the SD1.5 sizes, with the reference's
LoRA formula y = orig(x) + alpha * up(down(x)) injected, edlora.py:244-246): gradients of the NEW-CONCEPT EMBEDDING ROWS
(trainer_edlora.py:86-88, train_edlora.py:133-136) and of the 48 CLIPAttention LoRA pairs (:107-118).

Tolerances: bf16 operands, fp32 accumulation through 12 layers forward and backward: whole-gradient rel-L2 <= 3e-2 and
cosine >= 0.999 per parameter group (the UNet-side training test measures 8e-3 over a comparable depth)."""
import pytest
import torch

pytestmark = pytest.mark.gpu


def rel_l2(a, b):
    a, b = a.float().cpu(), b.float().cpu()
    return ((a - b).norm() / b.norm().clamp_min(1e-20)).item()


def _clip(layers):
    from transformers import CLIPTextConfig, CLIPTextModel
    cfg = CLIPTextConfig(vocab_size=49408 + 32, hidden_size=768, intermediate_size=3072, num_hidden_layers=layers,
                         num_attention_heads=12, max_position_embeddings=77)
    torch.manual_seed(0)
    return CLIPTextModel(cfg).eval()


def _ids(n_seq, concept_ids, g):
    ids = torch.randint(0, 49407, (n_seq, 77), generator=g)
    ids[:, 0] = 49406
    ids[:, 9:] = 49407
    for s in range(n_seq):            # two concept tokens per prompt (positions 4 and 5), layer-dependent ids
        ids[s, 4] = concept_ids[s % 16]
        ids[s, 5] = concept_ids[16 + s % 16]
    return ids


@pytest.mark.parametrize('layers,n_seq', [(2, 16), (12, 32)])
def test_clip_train_engine_vs_transformers_autograd(cuda, layers, n_seq):
    from mos_b200.clip_train_engine import CLIPTrainEngine
    from oracle import inject
    model = _clip(layers)
    sd = {k: v.clone() for k, v in model.state_dict().items()}
    lora = inject.random_lora_state(model, seed=7, where='CLIPAttention', up_std=0.05)
    alpha = 0.8
    concept_ids = list(range(49408, 49408 + 32))
    g = torch.Generator().manual_seed(3)
    ids = _ids(n_seq, concept_ids, g)
    dy = torch.randn(n_seq, 77, 768, generator=g) * 0.05
    # ---- reference: fp32 autograd through transformers with the reference's LoRA formula
    emb = model.get_input_embeddings().weight
    emb.requires_grad_(True)
    leaves = {k: v.clone().requires_grad_(True) for k, v in lora.items()}
    mods = dict(model.named_modules())
    for k in lora:
        if k.endswith('.lora_down.weight'):
            name = k[:-len('.lora_down.weight')]
            m = mods[name]

            def fwd(x, m=m, d=leaves[k], u=leaves[name + '.lora_up.weight'], orig=m.forward):
                return orig(x) + alpha * torch.nn.functional.linear(torch.nn.functional.linear(x, d), u)
            m.forward = fwd
    out_ref = model(ids)[0]
    (out_ref * dy).sum().backward()
    g_emb_ref = emb.grad[concept_ids]
    # ---- GPU engine
    eng = CLIPTrainEngine(sd, n_seq, lora=lora, lora_alpha=alpha, concept_token_ids=concept_ids)
    y = eng.forward_train(ids)
    e_fwd = rel_l2(y.view(n_seq, 77, 768), out_ref.detach())
    d_y = dy.reshape(-1, 768).to(cuda).to(torch.bfloat16).contiguous()
    eng.backward(d_y)
    torch.cuda.synchronize()
    e_emb = rel_l2(eng.emb_grad, g_emb_ref)
    cos_emb = torch.nn.functional.cosine_similarity(eng.emb_grad.flatten().cpu(), g_emb_ref.flatten(), dim=0).item()
    fg, fr, worst = [], [], (0.0, '')
    for m, (gd, gu) in eng.lora_grad_dict().items():
        for tag, a, b in (('down', gd, leaves[m + '.lora_down.weight'].grad), ('up', gu, leaves[m + '.lora_up.weight'].grad)):
            e = rel_l2(a, b)
            if e > worst[0]:
                worst = (e, f'{m}.{tag}')
            fg.append(a.flatten().cpu())
            fr.append(b.flatten())
    fg, fr = torch.cat(fg), torch.cat(fr)
    cos = torch.nn.functional.cosine_similarity(fg, fr, dim=0).item()
    print(f'CLIP train, {layers} layers x {n_seq} seqs: forward rel-L2 {e_fwd:.3e}; embedding-row grad rel-L2 {e_emb:.3e} '
          f'(cos {cos_emb:.5f}); LoRA grad ({fg.numel()} params) rel-L2 {rel_l2(fg, fr):.3e} (cos {cos:.5f}), worst '
          f'{worst[1]} {worst[0]:.3e}')
    assert e_fwd < 2e-2
    assert e_emb < 3e-2 and cos_emb > 0.999
    assert rel_l2(fg, fr) < 3e-2 and cos > 0.999
    assert worst[0] < 0.1
    # rows that are not concept tokens get no gradient slot; accumulate adds
    before = eng.emb_grad.clone()
    eng.backward(d_y, accumulate=True)
    torch.cuda.synchronize()
    assert rel_l2(eng.emb_grad, 2 * before) < 1e-3
    # checkpoint round trip in the reference's layout
    sd_l = eng.lora_state_dict()
    for k, v in lora.items():
        assert rel_l2(sd_l[k], v.reshape(sd_l[k].shape)) < 1e-6


def test_causal_attention_backward(cuda):
    """mos_attention_bwd(causal=1) vs autograd of F.scaled_dot_product_attention(is_causal=True): 12 heads of 64 dims run as
    head_dim 80 with zero pads, 77 tokens.  bf16 operands: rel-L2 <= 1.5e-2 per gradient."""
    import torch.nn.functional as F
    from mos_b200 import ops
    n_seq, H, n, d, dh = 4, 12, 77, 64, 80
    g = torch.Generator().manual_seed(0)
    q, k, v, do = (torch.randn(n_seq, H, n, d, generator=g).to(torch.bfloat16).float().requires_grad_(True) for _ in range(4))
    out = F.scaled_dot_product_attention(q, k, v, is_causal=True)
    out.backward(do.detach())
    BH, n8 = n_seq * H, 80

    def rows(t):
        r = torch.zeros(BH, n, 128, device=cuda, dtype=torch.bfloat16)
        r[..., :d] = t.detach().reshape(BH, n, d).to(cuda)
        return r
    Q, K, V, dO = rows(q), rows(k), rows(v), rows(do)
    Vt = torch.zeros(BH, dh, n8, device=cuda, dtype=torch.bfloat16)
    ops.heads_transpose(V, Vt)
    o = torch.zeros(n_seq, n, H * dh, device=cuda, dtype=torch.bfloat16)
    lse = torch.zeros(BH, n, device=cuda)
    ops.attention_causal(Q, K, Vt, o, batch=n_seq, heads=H, head_dim=dh, n=n, scale=d ** -0.5, lse2=lse)
    Qt, Kt, dOt = (torch.zeros(BH, dh, n8, device=cuda, dtype=torch.bfloat16) for _ in range(3))
    ops.heads_transpose(Q, Qt)
    ops.heads_transpose(K, Kt)
    ops.heads_transpose(dO, dOt)
    delta = torch.zeros(BH, n, device=cuda)
    ops.attn_delta(dO, o.view(n_seq * n, H * dh), delta, batch=n_seq, heads=H, head_dim=dh, N=n, ldo=H * dh)
    dqkv = torch.zeros(n_seq * n, 3 * H * dh, device=cuda, dtype=torch.bfloat16)
    Ca = H * dh
    ops.attention_bwd(Q, K, V, dO, Qt, Kt, dOt, lse, delta, dqkv[:, :Ca], dqkv[:, Ca:2 * Ca], dqkv[:, 2 * Ca:], batch=n_seq,
                      heads=H, head_dim=dh, nq=n, nk=n, scale=d ** -0.5, lddq=3 * Ca, lddk=3 * Ca, lddv=3 * Ca, causal=True)
    torch.cuda.synchronize()
    for s, (name, ref) in enumerate((('dq', q.grad), ('dk', k.grad), ('dv', v.grad))):
        got = dqkv[:, s * Ca:(s + 1) * Ca].reshape(n_seq, n, H, dh)[..., :d].permute(0, 2, 1, 3)
        e = rel_l2(got, ref)
        print(f'causal attention backward {name}: rel-L2 {e:.3e}')
        assert e < 1.5e-2
