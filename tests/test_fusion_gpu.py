"""Gradient fusion on the GPU (Gram-form L-BFGS, batched LoRA merge, engine-side Gram recording) vs the reference's
own `update_quasi_newton` / `merge_lora_into_weight` outputs stored in tests/golden/reference_golden.pt.

Tolerances: the optimiser is the same algorithm but the closure arithmetic differs (Gram form, fp32), so the
trajectories agree to rounding: relative Frobenius error of Wnew <= 2e-3 and final residual within 1 % (SURVEY §7.2.4).
"""
import os
import sys

import pytest
import torch

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'reference_golden.pt')


@pytest.fixture(scope='module')
def G():
    return torch.load(GOLD, weights_only=False)


def rel(a, b):
    a, b = a.float().cpu(), b.float().cpu()
    return ((a - b).norm() / b.norm().clamp_min(1e-30)).item()


def test_vector_primitives_and_sgemm(cuda):
    from mos_b200 import ops
    a, b = torch.randn(100003, device=cuda), torch.randn(100003, device=cuda)
    out, scratch = torch.zeros(1, device=cuda), torch.empty(256, device=cuda)
    ops.vec_dot(a, b, out, scratch)
    assert abs(out.item() - (a.double() @ b.double()).item()) < 1e-2
    ops.vec_absmax(a, out, scratch, 2.0)
    assert abs(out.item() - 2 * a.abs().max().item()) < 1e-5
    ops.vec_asum(a, out, scratch)
    assert abs(out.item() - a.abs().sum().item()) / a.abs().sum().item() < 1e-5
    y = b.clone()
    ops.vec_axpby(y, a, 0.5, 2.0)
    assert torch.allclose(y, 0.5 * a + 2 * b, atol=1e-5)
    A, B = torch.randn(321, 190, device=cuda), torch.randn(190, 257, device=cuda)
    C = torch.randn(321, 257, device=cuda)
    C0 = C.clone()
    ops.sgemm_nn(A, B, C, alpha=-1.0, beta=1.0)
    assert rel(C, C0 - A.double() @ B.double()) < 1e-5
    X, Y = torch.randn(45, 100, device=cuda), torch.randn(45, 37, device=cuda)
    g1, g2 = torch.empty(100, 100, device=cuda), torch.empty(100, 37, device=cuda)
    ops.gram_small(X, g1)
    ops.atb_small(X, Y, g2)
    assert rel(g1, X.double().t() @ X.double()) < 1e-5 and rel(g2, X.double().t() @ Y.double()) < 1e-5


@pytest.mark.parametrize('k', [0, 1, 7, 25])
@pytest.mark.parametrize('n', [245760, 100003])
def test_lbfgs_direction_bit_identical_to_host_recursion(cuda, k, n):
    """mos_lbfgs_direction (2k + 1 launches, coefficients on the device) vs the two-loop recursion driven from the host with
    vec_dot / vec_axpby exactly as gradient_fusion.lbfgs_minimize did before: same bits for d and <g, d>; twice in a row
    (the block counter must return to zero)."""
    from mos_b200 import ops
    gen = torch.Generator().manual_seed(7 + k)
    g = torch.randn(n, generator=gen).to(cuda)
    S = [(torch.randn(n, generator=gen) * 0.1).to(cuda) for _ in range(k)]
    Y = [(S[i] * (1.0 + 0.1 * i) + 0.05 * torch.randn(n, generator=gen).to(cuda)) for i in range(k)]
    scal, scratch = torch.zeros(1, device=cuda), torch.empty(256, device=cuda)

    def dot(a, b):
        ops.vec_dot(a, b, scal, scratch)
        return scal.item()

    rho = [1.0 / dot(Y[i], S[i]) for i in range(k)]
    h_diag = dot(Y[-1], S[-1]) / dot(Y[-1], Y[-1]) if k else 0.37
    # host-driven reference (the former code of lbfgs_minimize)
    al = [0.0] * k
    q = torch.empty_like(g)
    ops.vec_axpby(q, g, -1.0, 0.0)
    for i in range(k - 1, -1, -1):
        al[i] = dot(S[i], q) * rho[i]
        ops.vec_axpby(q, Y[i], -al[i], 1.0)
    ops.vec_axpby(q, q, h_diag, 0.0)
    for i in range(k):
        be = dot(Y[i], q) * rho[i]
        ops.vec_axpby(q, S[i], al[i] - be, 1.0)
    gtd_ref = dot(g, q)
    work = torch.zeros(64, device=cuda, dtype=torch.float64)
    partial = torch.zeros(260, device=cuda)
    gtd = torch.zeros(1, device=cuda)
    for rep in range(2):
        d = torch.full_like(g, float('nan'))
        ops.lbfgs_direction(S, Y, rho, g, h_diag, d, work, partial, gtd)
        torch.cuda.synchronize()
        assert torch.equal(d.view(torch.int32), q.view(torch.int32)), f'k={k} rep={rep}'
        assert gtd.item() == gtd_ref
        assert partial[256].item() == 0


@pytest.mark.parametrize('out_f,in_f,n_rows,iters', [(64, 96, 40, 30), (320, 768, 30, 60), (200, 130, 500, 25)])
def test_native_lbfgs_driver_bit_identical_to_python_driver(cuda, out_f, in_f, n_rows, iters):
    """csrc/lbfgs.cu (mos_lbfgs_solve_batch) issues the launches of gradient_fusion.lbfgs_minimize in the same order: the
    fused weight must be the same bits, for an under-determined (n < in) and an over-determined problem."""
    import gradient_fusion as gf
    g = torch.Generator().manual_seed(out_f + in_f)
    K = torch.randn(n_rows, in_f, generator=g).to(cuda)
    W0 = (torch.randn(out_f, in_f, generator=g) * in_f ** -0.5).to(cuda)
    Wt = W0 + 0.05 * torch.randn(out_f, in_f, generator=g).to(cuda)
    V = K @ Wt.t()
    G = (K.t() @ K).contiguous()
    Cm = (V.t() @ K).contiguous()
    vv = float((V.double() ** 2).sum())
    a = gf.solve_from_gram(G, Cm, vv, n_rows, W0, iters, native=False)
    b = gf.solve_from_gram(G, Cm, vv, n_rows, W0, iters, native=True)
    assert torch.equal(a.view(torch.int32), b.view(torch.int32))
    r0 = ((K @ W0.t() - V) ** 2).mean().item()
    r1 = ((K @ b.t() - V) ** 2).mean().item()
    assert r1 < 0.2 * r0
    # the batch entry with several workers: same bits again
    jobs = [(f'l{i}', G, Cm, vv, n_rows, W0, (out_f, in_f)) for i in range(5)]
    outs = gf.solve_all(jobs, iters, workers=3)
    for v in outs.values():
        assert torch.equal(v.view(torch.int32), a.cpu().view(torch.int32))


def test_dgemm_mixed_tilings(cuda):
    """the fp64 closure product in the default 64 x 64 tiling vs torch fp64 (MOS_DGEMM_TILE is read once per process;
    test_solver_engine_launches_gpu.py runs the 32 x 64 and 64 x 128 tiles in child processes)"""
    from mos_b200 import ops
    for M, K, N in ((320, 768, 768), (1280, 1280, 1280), (100, 70, 130)):
        A = torch.randn(M, K, device=cuda)
        B = torch.randn(K, N, device=cuda, dtype=torch.float64)
        C = torch.empty(M, N, device=cuda, dtype=torch.float64)
        ops.dgemm_mixed(A, B, C)
        ref = A.double() @ B
        assert ((C - ref).norm() / ref.norm()).item() < 1e-13


def test_gram_accumulate_tensor_core(cuda):
    from gradient_fusion import GramRecorder
    rec = GramRecorder(cuda)
    xs = [(torch.randn(1024, 320, device=cuda)).to(torch.bfloat16) for _ in range(3)]
    buf = torch.zeros(1024, 640, device=cuda, dtype=torch.bfloat16)
    for x in xs:
        buf[:, :320] = x
        rec('k', buf[:, :320], 1024, 320)           # strided view, as the engine hands it over
    ref = sum(x.double().t() @ x.double() for x in xs)
    assert rec.rows['k'] == 3072
    assert rel(rec.G['k'], ref) < 1e-5               # bf16 products are exact in fp32; only summation order differs


@pytest.mark.parametrize('case', ['', '2'])
def test_update_quasi_newton_vs_reference_golden(cuda, G, case):
    """same inputs as the reference run: K [30,64]/[400,48]; 50 L-BFGS iterations from W0."""
    from gradient_fusion import update_quasi_newton
    g = G['quasi_newton']
    K, V, W0, Wref = g['K' + case], g['V' + case], g['W0' + case], g['Wnew' + case]
    Wn = update_quasi_newton(K, V, W0.clone(), 50, 'cuda')
    res_ref = (K @ Wref.t() - V).norm().item()
    res_new = (K @ Wn.t() - V).norm().item()
    res_0 = (K @ W0.t() - V).norm().item()
    print(f'quasi-newton{case}: rel Frobenius vs reference {rel(Wn, Wref):.3e}; residual ours {res_new:.4e} '
          f'reference {res_ref:.4e} start {res_0:.4e}')
    assert rel(Wn, Wref) < 2e-3
    assert res_new <= res_ref * 1.01 + 1e-6 * res_0


def test_merge_lora_into_weight_vs_reference_golden(cuda, G):
    from gradient_fusion import merge_lora_into_weight
    m = G['merge_lora']
    out = merge_lora_into_weight(m['sd'], m['lora'], list(m['sd'].keys()), 'unet', m['alpha'], 'cuda')
    for k in m['sd']:
        assert rel(out[k], m['merged'][k]) < 1e-6 and out[k].shape == m['merged'][k].shape


def test_spatial_fusion_two_concepts_tiny(cuda):
    """merge_spatial_attention on the tiny topology: two synthetic ED-LoRAs; the fused weights must reproduce each
    concept's layer outputs on that concept's own features far better than the un-fused W0 does, and match an
    fp32 oracle solve (features recorded from the oracle UNet + reference-style L-BFGS) to bf16-feature accuracy."""
    from gradient_fusion import merge_spatial_attention
    from oracle import edlora_ref as er
    from oracle import inject
    from oracle import unet as ou
    from oracle.schedulers import DPMSolverMultistepScheduler
    u0 = ou.build_unet(0, ou.TINY)
    sd = {k: v.clone() for k, v in u0.state_dict().items()}
    loras = [inject.random_lora_state(u0, seed=10 + c, up_std=0.05) for c in range(2)]
    spatial = [{k: v for k, v in l.items() if 'attn2.to_k' not in k and 'attn2.to_v' not in k} for l in loras]
    embeds = [torch.randn(1, 16, 77, 768, generator=torch.Generator().manual_seed(20 + c)).to(torch.bfloat16).float()
              for c in range(2)]
    steps, iters, H = 3, 20, 16
    new_w = merge_spatial_attention(sd, spatial, [1.0, 1.0], embeds, iters, latent_hw=(H, H), num_inference_steps=steps,
                                    seed=0, block_out=ou.TINY['block_out_channels'], layers=1)
    assert len(new_w) == 4 * 6          # 4 transformer blocks x (attn1 q,k,v,out + attn2 q,out)
    # ---- oracle: record (input, output - bias) with hooks, as gradient_fusion.py:146-167 does, in fp32
    name = 'down_blocks.0.attentions.0.transformer_blocks.0.attn1.to_q'
    Xs, Vs = [], []
    for c in range(2):
        u = ou.build_unet(0, ou.TINY)
        inject.install_edlora_processors(u)
        inject.inject_lora(u, spatial[c], 1.0)
        mod = dict(u.named_modules())[name]
        rec = {'x': [], 'v': []}
        orig = mod.forward

        def hooked(x, orig=orig, rec=rec):
            y = orig(x)
            rec['x'].append(x.reshape(-1, x.shape[-1]))
            rec['v'].append(y.reshape(-1, y.shape[-1]))
            return y
        mod.forward = hooked
        sched = DPMSolverMultistepScheduler()
        sched.set_timesteps(steps)
        lat = torch.randn(1, 4, H, H, generator=torch.Generator().manual_seed(c))
        for t in sched.timesteps:
            with torch.no_grad():
                eps = u(lat, torch.tensor([int(t)]), embeds[c][:, :4]).sample
            lat = sched.step(eps, int(t), lat).prev_sample
        Xs.append(torch.cat(rec['x']))
        Vs.append(torch.cat(rec['v']))
    X, V = torch.cat(Xs), torch.cat(Vs)
    W0 = sd[name + '.weight']
    W_or = er.update_quasi_newton(X, V, W0, iters)
    Wn = new_w[name + '.weight']
    r0 = (X @ W0.t() - V).norm().item()
    r_or = (X @ W_or.t() - V).norm().item()
    r_new = (X @ Wn.t() - V).norm().item()
    print(f'spatial fusion {name}: residual W0 {r0:.4e} oracle {r_or:.4e} GPU {r_new:.4e}; '
          f'rel Frobenius vs oracle {rel(Wn, W_or):.3e}')
    assert r_new < 0.8 * r0                   # the fused weight explains both concepts better than W0
    assert r_new < 1.10 * r_or                # as well as the fp32 oracle solve (features are bf16 on the GPU)
    assert rel(Wn, W_or) < 2e-2


def test_text_encoder_fusion_two_concepts(cuda):
    """merge_text_encoder (gradient_fusion.py:460-565) on a 2-layer CLIP with two synthetic CLIPAttention LoRAs: the
    features come from the GPU CLIP engine on sequences padded to 77 (valid rows only), the oracle records them with
    forward hooks on transformers' CLIPTextModel run on the UN-padded sequences with the merged weights (as the reference
    does) and solves with the reference-style L-BFGS in fp32."""
    from transformers import CLIPTextConfig, CLIPTextModel
    from gradient_fusion import merge_text_encoder
    from oracle import edlora_ref as er
    from oracle import inject
    cfg = CLIPTextConfig(vocab_size=1000, hidden_size=768, intermediate_size=3072, num_hidden_layers=2,
                         num_attention_heads=12, max_position_embeddings=77, eos_token_id=999, bos_token_id=998,
                         pad_token_id=999)
    torch.manual_seed(0)
    base = CLIPTextModel(cfg).eval()
    sd = {k: v.clone() for k, v in base.state_dict().items()}
    loras = [inject.random_lora_state(base, seed=40 + c, where='CLIPAttention', up_std=0.05) for c in range(2)]
    alphas = [1.0, 0.7]
    g = torch.Generator().manual_seed(9)
    prompts = [[torch.cat([torch.tensor([998]), torch.randint(0, 990, (n,), generator=g), torch.tensor([999])])
                for n in (5, 2, 5, 2)] for _ in range(2)]
    iters = 30
    new_w = merge_text_encoder(sd, loras, alphas, prompts, iters, pad_id=999)
    assert len(new_w) == 2 * 4
    for name in ('text_model.encoder.layers.1.self_attn.q_proj.weight',
                 'text_model.encoder.layers.0.self_attn.out_proj.weight'):
        mod = name[:-len('.weight')]
        Xs, Vs = [], []
        for c in range(2):
            m = CLIPTextModel(cfg).eval()
            msd = {k: v.clone() for k, v in sd.items()}
            for k in list(loras[c]):
                if k.endswith('lora_down.weight'):
                    w = k.replace('.lora_down.weight', '.weight')
                    msd[w] = msd[w] + alphas[c] * loras[c][k.replace('lora_down', 'lora_up')] @ loras[c][k]
            m.load_state_dict(msd)
            rec = []
            h = dict(m.named_modules())[mod].register_forward_hook(
                lambda mod_, fin, fout, rec=rec: rec.append((fin[0].reshape(-1, 768), (fout - mod_.bias).reshape(-1, 768))))
            with torch.no_grad():
                for q in prompts[c]:
                    m(q.view(1, -1))
            h.remove()
            Xs.append(torch.cat([r[0] for r in rec]))
            Vs.append(torch.cat([r[1] for r in rec]))
        X, V = torch.cat(Xs), torch.cat(Vs)
        W0 = sd[name]
        W_or = er.update_quasi_newton(X, V, W0, iters)
        Wn = new_w[name]
        r0 = (X @ W0.t() - V).norm().item()
        r_or = (X @ W_or.t() - V).norm().item()
        r_new = (X @ Wn.t() - V).norm().item()
        print(f'text-encoder fusion {name}: residual W0 {r0:.4e} oracle {r_or:.4e} GPU {r_new:.4e}; '
              f'rel Frobenius vs oracle {rel(Wn, W_or):.3e}')
        # 44 rows against 768 unknowns per output: the oracle residual is ~0, so the GPU residual (bf16 features,
        # evaluated on the oracle's fp32 features) is bounded relative to the starting point instead
        assert r_new < 0.1 * r0
        assert rel(Wn, W_or) < 2e-2


def test_merge_kv_in_cross_attention_vs_reference_construction(cuda):
    """Config 3's cross-K/V stage: `merge_kv_in_cross_attention` (Gram form, one solve per layer) against the reference's
    own construction (gradient_fusion.py:394-455): per layer X = cat_c(features_c), V = cat_c(features_c @ merged_c^T),
    Wnew = update_quasi_newton(X, V, W0, iters) — run through the oracle port of `update_quasi_newton`, which is pinned
    to the reference's output by the golden test above.  3 concepts x 6 text positions (18 rows << 768 inputs:
    under-determined, exactly the reference's regime), two layers (K and V of one cross-attention, 320 x 768).
    Tolerances: fused weight rel-Frobenius <= 5e-4, the UPDATE (Wnew - W0) rel-Frobenius <= 5e-2 (the trajectory of a
    quasi-Newton iteration in Gram form rounds differently, SURVEY.md 7.2.4), final residual within 2 % of the reference's (or below 1e-5 of the starting residual: the system is under-determined and both solvers reach round-off)."""
    from gradient_fusion import merge_kv_in_cross_attention
    from oracle import edlora_ref as er
    g = torch.Generator().manual_seed(21)
    n_c, n_pos, C, D, iters = 3, 6, 320, 768, 200
    names = [(0, 'down_blocks.0.attentions.0.transformer_blocks.0.attn2.to_k.weight'),
             (0, 'down_blocks.0.attentions.0.transformer_blocks.0.attn2.to_v.weight'),
             (1, 'down_blocks.0.attentions.1.transformer_blocks.0.attn2.to_k.weight')]
    sd = {n: torch.randn(C, D, generator=g) * D ** -0.5 for _, n in names}
    feats = [{l: torch.randn(n_pos, D, generator=g) for l in (0, 1)} for _ in range(n_c)]
    tuned, alphas = [], [1.0, 0.7, 1.3]
    for c in range(n_c):
        t = {}
        for _, n in names:
            dn = n.replace('to_k.weight', 'to_k.lora_down.weight').replace('to_v.weight', 'to_v.lora_down.weight')
            t[dn] = torch.randn(4, D, generator=g) * D ** -0.5
            t[dn.replace('lora_down', 'lora_up')] = torch.randn(C, 4, generator=g) * 0.1
        tuned.append(t)
    new_w = merge_kv_in_cross_attention(sd, names, feats, tuned, alphas, iters, device='cuda')
    for layer_idx, n in names:
        dn = n.replace('to_k.weight', 'to_k.lora_down.weight').replace('to_v.weight', 'to_v.lora_down.weight')
        X = torch.cat([feats[c][layer_idx] for c in range(n_c)], 0)
        V = torch.cat([(((sd[n] + alphas[c] * tuned[c][dn.replace('lora_down', 'lora_up')] @ tuned[c][dn])
                         @ feats[c][layer_idx].T).T) for c in range(n_c)], 0)          # reference :403-429
        Wref = er.update_quasi_newton(X, V, sd[n].clone(), iters)
        Wn = new_w[n]
        r0 = (X @ sd[n].t() - V).norm().item()
        rr, rn = (X @ Wref.t() - V).norm().item(), (X @ Wn.t() - V).norm().item()
        e_w, e_d = rel(Wn, Wref), rel(Wn - sd[n], Wref - sd[n])
        print(f'cross-KV fusion {n.split(".")[-2]}[{layer_idx}]: W rel-Frob {e_w:.2e}, update rel-Frob {e_d:.2e}; residual '
              f'ours {rn:.3e} reference {rr:.3e} start {r0:.3e}')
        assert e_w < 5e-4 and e_d < 5e-2
        assert rn <= max(rr * 1.02, 1e-5 * r0)      # under-determined: both reach ~fp32 round-off of the start residual
