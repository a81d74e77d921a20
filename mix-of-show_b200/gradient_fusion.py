"""GPU gradient fusion — drop-in for the UNet half of the reference's `gradient_fusion.py`.

  update_quasi_newton(K_target, V_target, W, iters, device)     <- gradient_fusion.py:38-96 (+ chunk_compute_mse :22-35)
  merge_lora_into_weight(original, lora, layer_names, model_type, alpha, device)   <- :99-143
  merge_kv_in_cross_attention(...)   (text features supplied by the caller)          <- :325-457
  merge_spatial_attention(...)       (engine-side Gram recording instead of hooks)   <- :146-167, :579-624, :627-747

Design (DESIGN.md §4, fusion.cu header): the per-layer objective  mean((X W^T - V)^2)  depends on the recorded
features only through G = X^T X and C = V^T X.  The reference keeps X, V (GBs) in host RAM and re-streams them to the
GPU for each of the <= 62 closure evaluations per layer; here the UNet engine reduces the features to per-concept
Gram matrices on the fly (wgmma GEMM, fp32 accumulate), and a closure is one [out,in]x[in,in] fp32 GEMM.
The optimiser is the same algorithm the reference calls (torch.optim.LBFGS: history 25, lr 1, strong-Wolfe line
search, tolerance 1e-16, ONE .step of max_iter iterations, best iterate over all closure evaluations), restated here
over CUDA vector primitives (mos_vec_*), working on the correction D = W - W0 so that the quadratic is evaluated
without the cancellation of the raw Gram form.  The text-encoder half (merge_text_encoder) runs on the GPU CLIP engine
(mos_b200/clip_engine.py).  The reference's entry point (parse_new_concepts, merge_new_concepts_, get_text_feature,
compose_concepts and the CLI) is restated at the bottom of this file over those stages.
"""
import math
import os

import torch

from mos_b200 import ops
from mos_b200.dp import init_distributed

F32 = torch.float32


# ------------------------------------------------------------------------------------------------ L-BFGS (restated)
def _div(a, b):
    """a / b with IEEE semantics (a signed infinity or NaN for b = 0, where Python raises), as csrc/lbfgs.cu divides"""
    if b != 0 or b != b:
        return a / b
    return math.copysign(math.inf, a) * math.copysign(1.0, b) if a == a and a != 0 else math.nan


def _cubic_min(x1, f1, g1, x2, f2, g2, bounds=None):
    """Minimiser of the cubic through (x1,f1,g1), (x2,f2,g2), clipped to `bounds` (Nocedal & Wright eq. 3.59)."""
    lo, hi = bounds if bounds is not None else ((x1, x2) if x1 <= x2 else (x2, x1))
    d1 = g1 + g2 - _div(3.0 * (f1 - f2), x1 - x2)
    disc = d1 * d1 - g1 * g2
    if disc < 0:
        return 0.5 * (lo + hi)
    d2 = math.sqrt(disc)
    if x1 <= x2:
        pos = x2 - (x2 - x1) * _div(g2 + d2 - d1, g2 - g1 + 2.0 * d2)
    else:
        pos = x1 - (x1 - x2) * _div(g1 + d2 - d1, g1 - g2 + 2.0 * d2)
    return min(max(pos, lo), hi)


class _GramProblem:
    """f(D) = s <D, D G - 2 R> + f0,  grad = 2 s (D G - R);  D = W - W0 (flat fp32 on the device)."""

    def __init__(self, G, R, s, f0, W0):
        self.G, self.R, self.s, self.f0, self.W0 = G, R, float(s), float(f0), W0
        self.shape = tuple(R.shape)
        dev = R.device
        self.Y = torch.empty_like(R)          # fp64 [out, in]
        self.scal = torch.zeros(1, device=dev, dtype=F32)
        self.scratch = torch.empty(256, device=dev, dtype=F32)
        self.loss64 = torch.zeros(1, device=dev, dtype=torch.float64)
        self.scratch64 = torch.empty(256, device=dev, dtype=torch.float64)
        self.best_loss, self.best_D = float('inf'), None
        self.evals = 0
        # mos_lbfgs_direction: device coefficients, partial sums + block counter (zero between launches), <g, d>
        self.work = torch.zeros(64, device=dev, dtype=torch.float64)
        self.partial = torch.zeros(260, device=dev, dtype=F32)
        self.gtd = torch.zeros(1, device=dev, dtype=F32)
        self.scal2 = torch.zeros(2, device=dev, dtype=F32)

    def dot(self, a, b):
        ops.vec_dot(a, b, self.scal, self.scratch)
        return self.scal.item()

    def dot2(self, a, b, c, d):
        """(<a, b>, <c, d>) with one host synchronisation"""
        ops.vec_dot(a, b, self.scal2[0:1], self.scratch)
        ops.vec_dot(c, d, self.scal2[1:2], self.scratch)
        r = self.scal2.tolist()
        return r[0], r[1]

    def absmax2(self, a, b, scale_b):
        """(max |a|, max |scale_b b|) with one host synchronisation"""
        ops.vec_absmax(a, self.scal2[0:1], self.scratch, 1.0)
        ops.vec_absmax(b, self.scal2[1:2], self.scratch, scale_b)
        r = self.scal2.tolist()
        return r[0], r[1]

    def absmax(self, a, scale=1.0):
        ops.vec_absmax(a, self.scal, self.scratch, scale)
        return self.scal.item()

    def closure(self, D):
        """-> (loss float, grad tensor); tracks the best iterate like gradient_fusion.py:72-74."""
        ops.dgemm_mixed(D.view(self.shape), self.G, self.Y)
        grad = torch.empty_like(D)
        ops.ls_grad_loss(D, self.Y, self.R, self.s, self.f0, grad, self.loss64, self.scratch64)
        loss = self.loss64.item()
        self.evals += 1
        if math.isfinite(loss) and loss < self.best_loss:        # as csrc/lbfgs.cu: a non-finite loss never qualifies
            self.best_loss = loss
            self.best_D = D.clone()
        return loss, grad


def _strong_wolfe(P, x, t, d, f, g, gtd, c1=1e-4, c2=0.9, tol_change=1e-9, max_ls=25):
    """Strong-Wolfe line search (bracketing + zoom with cubic interpolation), as used by torch.optim.LBFGS."""
    d_norm = P.absmax(d)

    def phi(step):
        xt = x.clone()
        ops.vec_axpby(xt, d, step, 1.0)
        fv, gv = P.closure(xt)
        return fv, gv, P.dot(gv, d)

    f_new, g_new, gtd_new = phi(t)
    evals = 1
    t_prev, f_prev, g_prev, gtd_prev = 0.0, f, g, gtd
    done, it = False, 0
    br = None
    while it < max_ls:
        if f_new > f + c1 * t * gtd or (it > 1 and f_new >= f_prev):
            br = [[t_prev, f_prev, g_prev, gtd_prev], [t, f_new, g_new, gtd_new]]
            break
        if abs(gtd_new) <= -c2 * gtd:
            br = [[t, f_new, g_new, gtd_new]]
            done = True
            break
        if gtd_new >= 0:
            br = [[t_prev, f_prev, g_prev, gtd_prev], [t, f_new, g_new, gtd_new]]
            break
        lo, hi = t + 0.01 * (t - t_prev), t * 10.0
        t_next = _cubic_min(t_prev, f_prev, gtd_prev, t, f_new, gtd_new, bounds=(lo, hi))
        t_prev, f_prev, g_prev, gtd_prev = t, f_new, g_new, gtd_new
        t = t_next
        f_new, g_new, gtd_new = phi(t)
        evals += 1
        it += 1
    if it == max_ls:
        br = [[0.0, f, g, gtd], [t, f_new, g_new, gtd_new]]
    # zoom
    stalled = False
    if len(br) == 2:
        low, high = (0, 1) if br[0][1] <= br[1][1] else (1, 0)
    while not done and it < max_ls:
        if abs(br[1][0] - br[0][0]) * d_norm < tol_change:
            break
        t = _cubic_min(br[0][0], br[0][1], br[0][3], br[1][0], br[1][1], br[1][3])
        tmax, tmin = max(br[0][0], br[1][0]), min(br[0][0], br[1][0])
        eps = 0.1 * (tmax - tmin)
        if min(tmax - t, t - tmin) < eps:
            if stalled or t >= tmax or t <= tmin:
                t = tmax - eps if abs(t - tmax) < abs(t - tmin) else tmin + eps
                stalled = False
            else:
                stalled = True
        else:
            stalled = False
        f_new, g_new, gtd_new = phi(t)
        evals += 1
        it += 1
        if f_new > f + c1 * t * gtd or f_new >= br[low][1]:
            br[high] = [t, f_new, g_new, gtd_new]
            low, high = (0, 1) if br[0][1] <= br[1][1] else (1, 0)
        else:
            if abs(gtd_new) <= -c2 * gtd:
                done = True
            elif gtd_new * (br[high][0] - br[low][0]) >= 0:
                br[high] = list(br[low])
            br[low] = [t, f_new, g_new, gtd_new]
    sel = br[0] if len(br) == 1 else br[low]
    return sel[1], sel[2], sel[0], evals


def lbfgs_minimize(P, x0, max_iter, history=25, lr=1.0, tol_grad=1e-16, tol_change=1e-16):
    """ONE torch.optim.LBFGS.step(closure) with line_search_fn='strong_wolfe' (gradient_fusion.py:76-85)."""
    max_eval = max_iter * 5 // 4
    x = x0.clone()
    loss, g = P.closure(x)
    evals = 1
    if P.absmax(g) <= tol_grad:
        return x
    S, Y, rho = [], [], []          # curvature pairs (s_i = step, y_i = gradient change), rho_i = 1 / <y_i, s_i>
    h_diag, d, t, prev_g, prev_loss = 1.0, None, None, None, None
    n_iter = 0
    while n_iter < max_iter:
        n_iter += 1
        dev_gtd = False
        if n_iter == 1:
            d = g.clone()
            ops.vec_axpby(d, g, -1.0, 0.0)                      # d = -g
        else:
            y = g.clone()
            ops.vec_axpby(y, prev_g, -1.0, 1.0)                 # y = g - prev_g
            s = torch.empty_like(d)
            ops.vec_axpby(s, d, t, 0.0)                         # s = t d
            ys, yy = P.dot2(y, s, y, y)
            if ys > 1e-10:
                if len(S) == history:
                    S.pop(0), Y.pop(0), rho.pop(0)
                S.append(s), Y.append(y), rho.append(1.0 / ys)
                h_diag = ys / yy
            # two-loop recursion on q = -g, r = H0 q (one C-ABI call, 2k + 1 launches, coefficients stay on the device;
            # bit-identical to the recursion driven from here with vec_dot / vec_axpby), and <g, d> for the test below
            d = torch.empty_like(g)
            ops.lbfgs_direction(S, Y, rho, g, h_diag, d, P.work, P.partial, P.gtd)
            dev_gtd = True
        prev_g, prev_loss = g.clone(), loss
        if n_iter == 1:
            ops.vec_asum(g, P.scal, P.scratch)                  # |g|_1
            t = min(1.0, 1.0 / P.scal.item()) * lr
        else:
            t = lr
        gtd = P.gtd.item() if dev_gtd else P.dot(g, d)
        if gtd > -tol_change:
            break
        loss, g, t, ls_evals = _strong_wolfe(P, x, t, d, loss, g, gtd)
        ops.vec_axpby(x, d, t, 1.0)
        evals += ls_evals
        if n_iter == max_iter or evals >= max_eval:
            break
        g_max, step_max = P.absmax2(g, d, t)
        if g_max <= tol_grad or step_max <= tol_change or abs(loss - prev_loss) < tol_change:
            break
    return x


# ------------------------------------------------------------------------------------------------ solver front ends
def _gram_setup(G, Cm, vv, n_rows, W0):
    """one-time fp64 setup of a solve (like weight packing): residual right-hand side R = C - W0 G and f(W0); the Gram form
    squares the condition number, so the closure product D G is carried in fp64 on the device (mos_dgemm_mixed)"""
    out_f = Cm.shape[0]
    dev = Cm.device
    W0 = W0.to(dev, F32).contiguous()
    G = G.to(dev, F32).contiguous()
    s = 1.0 / (float(n_rows) * out_f)
    W0d, Gd, Cd = W0.double(), G.double().contiguous(), Cm.to(dev).double()
    Rd = (Cd - W0d @ Gd).contiguous()
    f0 = s * (float((W0d * (W0d @ Gd - 2.0 * Cd)).sum()) + float(vv))
    return W0, Gd, Rd, s, f0


# the L-BFGS loop runs in the library (csrc/lbfgs.cu); MOS_FUSION_NATIVE=0 selects the Python driver below, which issues the
# same launches in the same order (kept as the readable statement of the algorithm and as the yardstick of the tests)
FUSION_NATIVE = os.environ.get('MOS_FUSION_NATIVE', '1') != '0'


def solve_from_gram(G, Cm, vv, n_rows, W0, iters, native=None):
    """min_W (1/(n out)) (tr(W G W^T) - 2 tr(W C^T) + vv) by the reference's L-BFGS recipe, starting at W0.
    G [in,in], Cm [out,in] fp32 on the device; returns the best W over all closure evaluations (fp32, device)."""
    out_f, in_f = Cm.shape
    dev = Cm.device
    W0, Gd, Rd, s, f0 = _gram_setup(G, Cm, vv, n_rows, W0)
    if FUSION_NATIVE if native is None else native:
        best_D = torch.empty(out_f * in_f, device=dev, dtype=F32)
        ops.lbfgs_solve_batch([(Gd, Rd, s, f0, best_D)], iters, workers=1)
    else:
        P = _GramProblem(Gd, Rd, s, f0, W0)
        D0 = torch.zeros(out_f * in_f, device=dev, dtype=F32)
        lbfgs_minimize(P, D0, iters)
        best_D = P.best_D
        if best_D is None:
            raise ValueError('solve_from_gram: no closure evaluation gave a finite loss (G or R holds NaN or Inf)')
    Wn = W0.clone()
    ops.vec_axpby(Wn.view(-1), best_D, 1.0, 1.0)
    return Wn


FUSION_WORKERS = int(os.environ.get('MOS_FUSION_WORKERS', '8'))


def solve_all(jobs, iters, workers=None, to_host=True):
    """jobs: list of (name, G, Cm, vv, n_rows, W0, out_shape) - the independent per-layer problems of one fusion stage
    (gradient_fusion.py solves them one after the other, :394-455 / :518-563 / :690-745).  One L-BFGS solve is a chain of
    small kernels with a handful of host decisions per iteration and leaves the GPU mostly idle, so `workers` host threads
    drive `workers` solves at a time, each on its own CUDA stream.  Every solve runs exactly the arithmetic of the
    sequential code (results are bit-identical whatever the concurrency).  -> {name: fused weight (fp32, CPU; on the
    solving device with to_host=False)}."""
    workers = FUSION_WORKERS if workers is None else workers
    host = (lambda t: t.cpu()) if to_host else (lambda t: t)
    if not jobs:
        return {}
    dev = jobs[0][1].device
    out = {}
    if FUSION_NATIVE and dev.type == 'cuda':
        # host threads x CUDA streams inside the library (mos_lbfgs_solve_batch): no interpreter lock between the solves
        setups = [_gram_setup(G, Cm, vv, n, W0) for _, G, Cm, vv, n, W0, _ in jobs]
        bests = [torch.empty(W0.numel(), device=dev, dtype=F32) for W0, *_ in setups]
        ops.lbfgs_solve_batch([(Gd, Rd, s, f0, b) for (W0, Gd, Rd, s, f0), b in zip(setups, bests)], iters, workers=workers)
        for (name, *_, shape), (W0, *_), b in zip(jobs, setups, bests):
            Wn = W0.clone()
            ops.vec_axpby(Wn.view(-1), b, 1.0, 1.0)
            out[name] = host(Wn.reshape(shape))
        return out
    if workers <= 1 or len(jobs) == 1 or dev.type != 'cuda':
        for name, G, Cm, vv, n, W0, shape in jobs:
            out[name] = host(solve_from_gram(G, Cm, vv, n, W0, iters).reshape(shape))
        return out
    import queue
    import threading
    torch.cuda.synchronize(dev)                 # the Gram matrices / right-hand sides were built on the caller's stream
    # largest problems first: the tail of the schedule is then filled with short solves
    order = sorted(range(len(jobs)), key=lambda i: -jobs[i][2].numel())
    todo = queue.SimpleQueue()
    for i in order:
        todo.put(i)
    errors, results = [], {}

    def run():
        stream = torch.cuda.Stream(device=dev)
        try:
            with torch.cuda.device(dev), torch.cuda.stream(stream):
                while True:
                    try:
                        i = todo.get_nowait()
                    except queue.Empty:
                        break
                    name, G, Cm, vv, n, W0, shape = jobs[i]
                    results[name] = solve_from_gram(G, Cm, vv, n, W0, iters).reshape(shape)
                stream.synchronize()
        except BaseException as exc:            # re-raised in the caller's thread
            errors.append(exc)

    threads = [threading.Thread(target=run, daemon=True) for _ in range(min(workers, len(jobs)))]
    for t in threads:
        t.start()
    for t in threads:
        t.join()
    if errors:
        raise errors[0]
    torch.cuda.synchronize(dev)
    return {job[0]: host(results[job[0]]) for job in jobs}


def update_quasi_newton(K_target, V_target, W, iters, device='cuda'):
    """Reference signature (gradient_fusion.py:38): K [n,in], V [n,out], W [out,in] (or 1x1-conv 4-D) -> Wnew."""
    shape = W.shape
    W2 = W.detach().reshape(shape[0], -1)
    if K_target.ndim == 4:                                     # 1x1 conv features [n, in, h, w] (:66-68)
        K_target = K_target.permute(0, 2, 3, 1).reshape(-1, K_target.shape[1])
        V_target = V_target.permute(0, 2, 3, 1).reshape(-1, V_target.shape[1])
    K = K_target.detach().to(device, F32).contiguous()
    V = V_target.detach().to(device, F32).contiguous()
    n, d_in = K.shape
    G = torch.empty(d_in, d_in, device=device, dtype=F32)
    Cm = torch.empty(V.shape[1], d_in, device=device, dtype=F32)
    ops.gram_small(K, G)
    ops.atb_small(V, K, Cm)
    scal, scratch = torch.zeros(1, device=device), torch.empty(256, device=device)
    ops.vec_dot(V.view(-1), V.view(-1), scal, scratch)
    Wn = solve_from_gram(G, Cm, scal.item(), n, W2, iters)
    return Wn.reshape(shape).cpu()


def merge_lora_into_weight(original_state_dict, lora_state_dict, modification_layer_names, model_type, alpha, device):
    """W' = W + alpha * up @ down for every listed layer that has a LoRA pair (gradient_fusion.py:99-143), one
    batched kernel launch for all layers."""
    assert model_type in ['unet', 'text_encoder']
    subs = (('q_proj', 'k_proj', 'v_proj', 'out_proj', 'fc1', 'fc2') if model_type == 'text_encoder' else
            ('to_q', 'to_k', 'to_v', 'to_out.0', 'ff.net.0.proj', 'ff.net.2', 'proj_out', 'proj_in'))
    new_sd = {k: v.clone() for k, v in original_state_dict.items()}
    rows, keep = [], []
    for k in modification_layer_names:
        down_name = k
        for sname in subs:
            down_name = down_name.replace(f'{sname}.weight', f'{sname}.lora_down.weight')
        up_name = down_name.replace('lora_down', 'lora_up')
        if up_name not in lora_state_dict:
            continue
        Wd = new_sd[k].to(device, F32).contiguous()
        dn = lora_state_dict[down_name].to(device, F32).contiguous()
        up = lora_state_dict[up_name].to(device, F32).contiguous()
        out_f, rank = up.shape[0], dn.shape[0]
        rows.append([Wd.data_ptr(), dn.data_ptr(), up.data_ptr(), out_f, Wd.numel() // out_f, rank])
        keep.append((k, Wd, dn, up))
    if rows:
        table = torch.tensor(rows, dtype=torch.int64, device=device)
        ops.lora_merge(table, len(rows), float(alpha))
        for k, Wd, _, _ in keep:
            new_sd[k] = Wd.to(original_state_dict[k].dtype).reshape(original_state_dict[k].shape)
    return new_sd


def _merged(W0, down, up, alpha, device):
    """W0 + alpha * up @ down through the batched merge kernel."""
    Wc = W0.to(device, F32).clone().contiguous()
    dn = down.to(device, F32).reshape(down.shape[0], -1).contiguous()
    u = up.to(device, F32).reshape(up.shape[0], -1).contiguous()
    table = torch.tensor([[Wc.data_ptr(), dn.data_ptr(), u.data_ptr(), u.shape[0], dn.shape[1], dn.shape[0]]],
                         dtype=torch.int64, device=device)
    ops.lora_merge(table, 1, float(alpha))
    torch.cuda.current_stream().synchronize()      # dn / u are temporaries of this call
    return Wc


def lora_weight_names(lora_list):
    """sorted '<module>.weight' names of every layer some LoRA of `lora_list` touches: the weights a stage solves"""
    return sorted({k.replace('.lora_down', '').replace('.lora_up', '') for t in lora_list for k in t})


def _owned(names, solve_names):
    """the names this call solves (all of them for solve_names=None), in the stage's own order"""
    if solve_names is None:
        return names
    own = set(solve_names)
    return [n for n in names if n in own]


def merge_kv_in_cross_attention(unet_state_dict, cross_kv_layer_names, text_features, unet_crosskv_list, alphas,
                                optimize_iters, device='cuda', solve_names=None):
    """Cross-attention K/V fusion (gradient_fusion.py:325-457).  text_features[c][layer_idx] = CLIP features of
    concept c at its concept-token (+EOS) positions [n_pos, 768] (gradient_fusion.py:182-199; CLIP runs upstream).
    cross_kv_layer_names: [(layer_idx, 'down_blocks....attn2.to_k.weight'), ...] in the reference's order.
    solve_names: solve (and return, still on the device) only these weights - one rank's share of a sharded fusion
    (fusion_plan); every weight is bit-identical to the same weight of the full call."""
    jobs = []
    own = None if solve_names is None else set(solve_names)
    for layer_idx, name in cross_kv_layer_names:
        if own is not None and name not in own:
            continue
        W0 = unet_state_dict[name].to(device, F32)
        d_in = W0.shape[1]
        G = torch.zeros(d_in, d_in, device=device)
        Cm = torch.zeros(W0.shape[0], d_in, device=device)
        vv, n = 0.0, 0
        dn_name = name.replace('to_k.weight', 'to_k.lora_down.weight').replace('to_v.weight', 'to_v.lora_down.weight')
        for c, tuned in enumerate(unet_crosskv_list):
            X = text_features[c][layer_idx].to(device, F32).contiguous()
            Wc = _merged(W0, tuned[dn_name], tuned[dn_name.replace('lora_down', 'lora_up')], alphas[c], device)  # :403-409
            Gc = torch.empty(d_in, d_in, device=device)
            ops.gram_small(X, Gc)
            WG = torch.empty_like(Cm)
            ops.sgemm_nn(Wc.contiguous(), Gc, WG)
            ops.vec_axpby(G.view(-1), Gc.view(-1), 1.0, 1.0)
            ops.vec_axpby(Cm.view(-1), WG.view(-1), 1.0, 1.0)
            vv += float((Wc.double() * WG.double()).sum())
            n += X.shape[0]
        jobs.append((name, G, Cm, vv, n, W0, tuple(W0.shape)))
    return solve_all(jobs, optimize_iters, to_host=solve_names is None)


class _RowRecorder:
    """CLIPTextEngine hook for the text-encoder fusion: keeps the rows of the valid (un-padded) token positions of
    every recorded GEMM input as fp32 (a few hundred rows of 768 / 3072: no tensor-core Gram needed).
    keys: the record keys some solve uses (None: all)."""

    def __init__(self, rows, heads, d, dh, keys=None):
        self.rows, self.heads, self.d, self.dh, self.keys = rows, heads, d, dh, keys
        self.X = {}

    def __call__(self, key, A, M, C):
        if self.keys is not None and key not in self.keys:
            return
        X = A[self.rows].float()
        if C == self.heads * self.dh and self.dh != self.d:       # attention output in the padded head layout
            X = X.view(-1, self.heads, self.dh)[:, :, :self.d].reshape(-1, self.heads * self.d)
        self.X[key] = X.contiguous()


# module suffix of a fused weight -> suffix of the engine record key of its input (q|k|v share one input).  UNet keys are
# relative to the Transformer2DModel ('...attentions.{j}': proj_in / proj_out) or its transformer_blocks.0 (the rest);
# CLIP keys to 'text_model.encoder.layers.{i}'.  attn2.to_k / to_v read the text embeddings: merge_kv_in_cross_attention.
RECORD_KEYS = (('.attn1.to_q', '.attn1.in'), ('.attn1.to_k', '.attn1.in'), ('.attn1.to_v', '.attn1.in'),
               ('.attn1.to_out.0', '.attn1.to_out.0'), ('.attn2.to_q', '.attn2.to_q'),
               ('.attn2.to_out.0', '.attn2.to_out.0'), ('.ff.net.0.proj', '.ff.net.0.proj'), ('.ff.net.2', '.ff.net.2'),
               ('.proj_in', '.proj_in'), ('.proj_out', '.proj_out'),
               ('.self_attn.q_proj', '.self_attn.in'), ('.self_attn.k_proj', '.self_attn.in'),
               ('.self_attn.v_proj', '.self_attn.in'), ('.self_attn.out_proj', '.self_attn.out_proj'),
               ('.mlp.fc1', '.mlp.fc1'), ('.mlp.fc2', '.mlp.fc2'))


def record_key(name):
    """'<module>.weight' of a spatial UNet or a CLIP linear -> the key under which the engine records its input, e.g.
    '...transformer_blocks.0.attn1.to_k.weight' -> '...transformer_blocks.0.attn1.in'."""
    mod = name[:-len('.weight')] if name.endswith('.weight') else name
    for leaf, key in RECORD_KEYS:
        if mod.endswith(leaf):
            return mod[:-len(leaf)] + key
    raise KeyError(f'{name}: no recorded input for this layer in gradient fusion')


def merge_text_encoder(text_state_dict, text_encoder_list, alphas, prompt_ids, optimize_iters, device='cuda',
                       pad_id=49407, solve_names=None):
    """Text-encoder fusion (gradient_fusion.py:460-565).  text_encoder_list[c]: concept c's CLIP LoRA
    ({'text_model.encoder.layers.{i}.self_attn.{q,k,v,out}_proj.lora_{down,up}.weight'}, with `where: CLIPEncoderLayer`
    also '...layers.{i}.mlp.fc{1,2}.lora_{down,up}.weight'); prompt_ids[c]: the un-padded
    token-id sequences of concept c's 32 layer-bound prompts ('photo of a <c>' and '<c>' x 16, :515-520; the tokenizer
    runs upstream).  For every concept its LoRA is merged (:505-512), the prompts run through the GPU CLIP engine and
    the inputs of the LoRA'd linears at ALL valid token positions are recorded (the reference's forward hooks, :146-167,
    :525-541); every layer is then solved from the accumulated Gram matrices as in merge_kv_in_cross_attention.
    Causal attention makes the features of a valid position independent of the padding behind it, so the sequences are
    padded to 77 for the engine and only the valid rows are kept.  solve_names: as merge_kv_in_cross_attention; only
    the inputs of these weights are recorded, and nothing runs when there are none."""
    from mos_b200.clip_engine import CLIPTextEngine
    names = _owned(lora_weight_names(text_encoder_list), solve_names)
    if not names:
        return {}
    keys = {record_key(n) for n in names}
    feats = []
    for c, tuned in enumerate(text_encoder_list):
        seqs = [torch.as_tensor(p_).reshape(-1) for p_ in prompt_ids[c]]
        n_seq = len(seqs)
        eng = CLIPTextEngine(text_state_dict, n_seq, lora=tuned, lora_alpha=alphas[c], merge_lora=True, device=device)
        ids = torch.full((n_seq, eng.T), pad_id, dtype=torch.long)
        rows = []
        for s_, q in enumerate(seqs):
            assert 0 < q.numel() <= eng.T
            ids[s_, :q.numel()] = q
            rows += [s_ * eng.T + t for t in range(q.numel())]
        rec = _RowRecorder(torch.tensor(rows, device=device), eng.heads, eng.d, eng.dh, keys)
        eng.gram_rec = rec
        eng(ids)
        feats.append(rec.X)
    jobs = []
    for name in names:                                       # e.g. 'text_model.encoder.layers.0.self_attn.q_proj.weight'
        mod = name[:-len('.weight')]
        rec_key = record_key(name)
        W0 = text_state_dict[name].to(device, F32)
        d_in = W0.shape[1]
        G = torch.zeros(d_in, d_in, device=device)
        Cm = torch.zeros(W0.shape[0], d_in, device=device)
        vv, n = 0.0, 0
        for c, tuned in enumerate(text_encoder_list):
            X = feats[c][rec_key]
            Wc = _merged(W0, tuned[mod + '.lora_down.weight'], tuned[mod + '.lora_up.weight'], alphas[c], device) \
                if (mod + '.lora_down.weight') in tuned else W0
            Gc = torch.empty(d_in, d_in, device=device)
            ops.gram_small(X, Gc)
            WG = torch.empty_like(Cm)
            ops.sgemm_nn(Wc.contiguous(), Gc, WG)
            ops.vec_axpby(G.view(-1), Gc.view(-1), 1.0, 1.0)
            ops.vec_axpby(Cm.view(-1), WG.view(-1), 1.0, 1.0)
            vv += float((Wc.double() * WG.double()).sum())
            n += X.shape[0]
        jobs.append((name, G, Cm, vv, n, W0, tuple(W0.shape)))
    return solve_all(jobs, optimize_iters, to_host=solve_names is None)


class GramRecorder:
    """Engine-side replacement of the reference's forward hooks (gradient_fusion.py:146-167): instead of copying
    every (input, output - bias) pair to host RAM, accumulate G += X^T X per recorded GEMM input on the tensor
    cores (transpose -> wgmma GEMM with fp32 accumulate output).  keys: the record keys some solve uses (None: all); an
    attention-only fusion then issues no Gram launch for the feed-forward / proj_in / proj_out inputs (ff.net.2: 5120^2)."""

    def __init__(self, device, keys=None):
        self.dev, self.G, self.rows, self._xt, self.keys = device, {}, {}, {}, keys

    def __call__(self, key, A, M, C):
        if self.keys is not None and key not in self.keys:
            return
        G = self.G.get(key)
        first = G is None
        if first:
            G = self.G[key] = torch.zeros(C, C, device=self.dev, dtype=F32)
            self.rows[key] = 0
        xt = self._xt.get((C, M, A.dtype))
        if xt is None:
            xt = self._xt[(C, M, A.dtype)] = torch.empty(C, M, device=self.dev, dtype=A.dtype)
        ops.transpose_bf16(A, xt, rows=M, C=C, ldx=A.stride(0))
        ops.gemm(xt, xt, G, out_f32=True, accumulate=True)
        self.rows[key] += M


def merge_spatial_attention(unet_state_dict, unet_spatial_attn_list, alphas, concept_embeds, optimize_iters,
                            latent_hw=(64, 64), num_inference_steps=20, seed=0, device='cuda', block_out=None,
                            layers=None, solve_names=None):
    """Spatial-attention fusion (gradient_fusion.py:627-747).  concept_embeds[c] = layer-wise prompt embeddings
    [1,16,77,768] of 'photo of a <concept c>' (CLIP runs upstream).  For every concept: merge its LoRA, run the
    20-step DPM-Solver++ sampling (batch 1, no CFG, all steps recorded, :579-624) on the engine with the Gram
    recorder, then solve every LoRA'd layer from the accumulated Gram matrices.  Besides the attention projections this
    covers the `where: Transformer2DModel` layers (proj_in / proj_out as 1x1 convs, returned 4-D; ff.net.0.proj solved in
    the state-dict row order, ff.net.2).  solve_names: as merge_text_encoder (every concept's sampling still runs in full
    when some are given: the recorded inputs depend on the whole UNet)."""
    from mos_b200.engine import UNetEngine, ehs_to_layer_major
    from mos_b200.scheduler import DPMSolverPP2M
    H, Wd = latent_hw
    kw = {}
    if block_out is not None:
        kw = dict(block_out=block_out, layers=layers)
    names = _owned(lora_weight_names(unet_spatial_attn_list), solve_names)
    if not names:
        return {}
    keys = {record_key(n) for n in names}
    grams, merged_w = [], []
    eng = None
    prof = os.environ.get('MOS_FUSION_PROFILE') == '1'       # stage timing printout (tools/config_bench.py)
    import time
    marks = []

    def mark(label):
        if prof:
            torch.cuda.synchronize()
            marks.append((label, time.perf_counter()))

    mark('start')
    for c, tuned in enumerate(unet_spatial_attn_list):
        mark(f'concept {c}: pack')
        if eng is None:
            eng = UNetEngine(unet_state_dict, 1, H, Wd, lora=tuned, lora_alpha=alphas[c], merge_lora=True, device=device,
                             use_graph=False, **kw)
        else:
            eng.set_merged_lora(tuned, alphas[c], state_dict=unet_state_dict)   # only the LoRA'd projections are re-packed
        rec = GramRecorder(device, keys)
        eng.gram_rec = rec
        nx = len(eng.xattn_names)
        sched = DPMSolverPP2M()
        sched.set_timesteps(num_inference_steps)
        g = torch.Generator(device='cpu').manual_seed(seed + c)
        latents = torch.randn(1, 4, H, Wd, generator=g).to(device)
        x0_prev = torch.zeros_like(latents)
        eng.in_ehs.copy_(ehs_to_layer_major(concept_embeds[c].to(device), nx))
        eng.in_latents.copy_(latents)
        mark(f'concept {c}: forwards')
        for i, t in enumerate(sched.timesteps):
            eng.in_t.fill_(float(t))
            eng.run()
            ops.cfg_dpmpp_step(eng.out_eps, latents, x0_prev, eng.in_latents.view(-1), cfg=False, guidance=1.0,
                               coef=sched.coefficients(i))
        grams.append(rec)
        merged_w.append(tuned)
        eng.gram_rec = None
    mark('job assembly')
    jobs = []
    for name in names:                                          # e.g. '...attn1.to_q.weight'
        mod = name[:-len('.weight')]
        rec_key = record_key(name)
        W0 = unet_state_dict[name].to(device, F32).reshape(unet_state_dict[name].shape[0], -1)
        d_in = W0.shape[1]
        G = torch.zeros(d_in, d_in, device=device)
        Cm = torch.zeros(W0.shape[0], d_in, device=device)
        vv, n = 0.0, 0
        for c, tuned in enumerate(unet_spatial_attn_list):
            Gc = grams[c].G[rec_key]
            Wc = _merged(W0, tuned[mod + '.lora_down.weight'], tuned[mod + '.lora_up.weight'], alphas[c], device) \
                if (mod + '.lora_down.weight') in tuned else W0
            WG = torch.empty_like(Cm)
            ops.sgemm_nn(Wc.contiguous(), Gc, WG)
            ops.vec_axpby(G.view(-1), Gc.view(-1), 1.0, 1.0)
            ops.vec_axpby(Cm.view(-1), WG.view(-1), 1.0, 1.0)
            vv += float((Wc.double() * WG.double()).sum())
            n += grams[c].rows[rec_key]
        jobs.append((name, G, Cm, vv, n, W0, tuple(unet_state_dict[name].shape)))
    mark('solve')
    out = solve_all(jobs, optimize_iters, to_host=solve_names is None)
    mark('end')
    if prof:
        agg = {}
        for (label, t0), (_, t1) in zip(marks[:-1], marks[1:]):
            key = label.split(': ')[-1]
            agg[key] = agg.get(key, 0.0) + (t1 - t0)
        print('merge_spatial_attention seconds: ' + ', '.join(f'{k} {v:.2f}' for k, v in agg.items()), flush=True)
    return out


# ------------------------------------------------------------------------------------------------ orchestration (host)
# The reference's entry point (gradient_fusion.py:750-851): checkpoint parsing, tokenizer / embedding-table bookkeeping,
# prompt construction and the order of the three fusion stages, restated over the feature-level stage functions above and
# this repo's model containers.  Pure host logic; the arithmetic lives in the stage functions.
TEMPLATE_SIMPLE = 'photo of a {}'                      # gradient_fusion.py:19
NUM_CROSS_ATTENTION_LAYERS = 16


# the layers the fusion stages solve (the reference's candidate lists, gradient_fusion.py:482-488 / :637-645)
_UNET_LORA_SUFFIXES = tuple(f'.{m}.lora_{d}.weight'
                            for m in [f'{a}.{p}' for a in ('attn1', 'attn2') for p in ('to_q', 'to_k', 'to_v', 'to_out.0')]
                            + ['ff.net.0.proj', 'ff.net.2', 'proj_in', 'proj_out'] for d in ('down', 'up'))
_TEXT_LORA_SUFFIXES = tuple(f'.{m}.lora_{d}.weight' for m in ('self_attn.q_proj', 'self_attn.k_proj', 'self_attn.v_proj',
                                                               'self_attn.out_proj', 'mlp.fc1', 'mlp.fc2')
                            for d in ('down', 'up'))


def _check_lora_targets(params, path):
    """The fusion stages cover the reference's LoRA placements: `where: Attention` / `Transformer2DModel` in the UNet
    (attention projections, ff.net, proj_in / proj_out) and `where: CLIPAttention` / `CLIPEncoderLayer` in the text encoder
    (self_attn projections, mlp.fc1 / fc2).  A LoRA anywhere else (e.g. on a resnet conv) is refused HERE, before any stage
    has run, instead of failing with a KeyError half way through the fusion."""
    bad = [k for k in (params.get('unet') or {}) if not k.endswith(_UNET_LORA_SUFFIXES)]
    bad += [k for k in (params.get('text_encoder') or {}) if not k.endswith(_TEXT_LORA_SUFFIXES)]
    if bad:
        raise ValueError(f'{path}: unsupported LoRA target(s) {bad[:3]}{" ..." if len(bad) > 3 else ""}: gradient fusion '
                         'handles LoRA on the transformer blocks (where: Attention / Transformer2DModel) and the CLIP encoder '
                         'layers (where: CLIPAttention / CLIPEncoderLayer) only')


def parse_new_concepts(concept_cfg):
    """gradient_fusion.py:262-322: split every concept's `.pth` into embedding / text-encoder / cross-K/V / spatial parts.
    A concept embedding without 16 rows (a vanilla LoRA checkpoint) is refused here, naming the file."""
    import json
    if isinstance(concept_cfg, str):
        with open(concept_cfg, 'r') as f:
            concept_list = json.load(f)
    else:
        concept_list = concept_cfg
    embedding_list, text_encoder_list, unet_crosskv_list, unet_spatial_attn_list = [], [], [], []
    crosskv_matches = ['attn2.to_k.lora', 'attn2.to_v.lora']
    for concept in concept_list:
        model = torch.load(concept['lora_path'], map_location='cpu')['params']
        _check_lora_targets(model, concept['lora_path'])
        emb = model.get('new_concept_embedding')
        for name, e in (emb or {}).items():
            if e.shape[0] != NUM_CROSS_ATTENTION_LAYERS:
                raise ValueError(f"{concept['lora_path']}: the embedding of {name} has {e.shape[0]} rows, gradient fusion "
                                 f'takes ED-LoRA checkpoints ({NUM_CROSS_ATTENTION_LAYERS} layer-wise rows per concept); '
                                 'a vanilla LoRA (enable_edlora: false) cannot be fused')
        embedding_list.append(emb if emb is not None and len(emb) != 0 else None)
        te = model.get('text_encoder')
        text_encoder_list.append(te if te is not None and len(te) != 0 else None)
        if 'unet' in model and len(model['unet']) != 0:
            kv = {k: v for k, v in model['unet'].items() if any(x in k for x in crosskv_matches)}
            sp = {k: v for k, v in model['unet'].items() if all(x not in k for x in crosskv_matches)}
            unet_crosskv_list.append(kv if len(kv) != 0 else None)
            unet_spatial_attn_list.append(sp if len(sp) != 0 else None)
        else:
            unet_crosskv_list.append(None)
            unet_spatial_attn_list.append(None)
    return embedding_list, text_encoder_list, unet_crosskv_list, unet_spatial_attn_list, concept_list


def merge_new_concepts_(embedding_list, concept_list, tokenizer, text_encoder):
    """gradient_fusion.py:214-259: 16 new tokens `<new{k}>` per `<concept>` word (numbered consecutively over all
    concepts), embedding table resized and the learned rows written; returns (embedding_features, new_concept_cfg)."""
    embedding_features, new_concept_cfg = {}, {}
    start_idx = 0
    for embedding, concept in zip(embedding_list, concept_list):
        for concept_name in concept['concept_name'].split(' '):
            if not concept_name.startswith('<'):
                continue
            assert concept_name in embedding, 'check the config, the provide concept name is not in the lora model'
            new_token_names = [f'<new{start_idx + layer_id}>' for layer_id in range(NUM_CROSS_ATTENTION_LAYERS)]
            num_added_tokens = tokenizer.add_tokens(new_token_names)
            assert num_added_tokens == NUM_CROSS_ATTENTION_LAYERS
            new_token_ids = [tokenizer.convert_tokens_to_ids(n) for n in new_token_names]
            text_encoder.resize_token_embeddings(len(tokenizer))
            token_embeds = text_encoder.get_input_embeddings().weight.data
            token_embeds[new_token_ids] = embedding[concept_name].to(token_embeds.device, token_embeds.dtype)
            embedding_features[concept_name] = embedding[concept_name]
            start_idx += NUM_CROSS_ATTENTION_LAYERS
            new_concept_cfg[concept_name] = {'concept_token_ids': new_token_ids, 'concept_token_names': new_token_names}
    return embedding_features, new_concept_cfg


def _unpadded_ids(text, tokenizer):
    return tokenizer(text, truncation=True, max_length=tokenizer.model_max_length, return_length=True,
                     return_overflowing_tokens=False, padding='do_not_pad').input_ids


@torch.no_grad()
def get_text_feature(prompts, tokenizer, text_encoder, device, return_type='category_embedding', eos_id=49407):
    """gradient_fusion.py:182-211.  'category_embedding': features at the positions whose token id is >= eos_id (the new
    concept tokens AND the end token, :196-197) of every un-padded prompt, concatenated; 'full_embedding': [n, 77, 768]."""
    if return_type == 'category_embedding':
        feats = []
        for text in prompts:
            tokens = _unpadded_ids(text, tokenizer)
            pos = torch.where(torch.tensor(tokens) >= eos_id)[0]
            h = text_encoder(torch.LongTensor(tokens).reshape(1, -1).to(device))[0]
            feats.append(h[:, pos.to(h.device)].reshape(-1, h.shape[-1]))
        return torch.cat(feats, 0).float()
    if return_type == 'full_embedding':
        ids = tokenizer(prompts, padding='max_length', max_length=tokenizer.model_max_length, truncation=True,
                        return_tensors='pt').input_ids
        return text_encoder(ids.to(device))[0]
    raise NotImplementedError(return_type)


def cross_kv_layer_names(unet):
    """[(cross_attention_idx, '<...>.attn2.to_k.weight'), (idx, '<...>.to_v.weight'), ...] in the reference's
    down -> mid -> up parameter order (gradient_fusion.py:331-369)."""
    names, idx = [], -1
    for prefix, block in (('down_blocks.', unet.down_blocks), ('mid_block.', unet.mid_block), ('up_blocks.', unet.up_blocks)):
        for name, _ in block.named_parameters():
            if 'attn2.to_k' in name:
                idx += 1
                names.append((idx, prefix + name))
                names.append((idx, prefix + name.replace('to_k', 'to_v')))
    return names


# ------------------------------------------------------------------------------------------------ sharding across ranks
def solve_cost(shape, iters):
    """planned cost of one layer solve: out * in^2 * iters, the fp64 closure GEMM D G of every L-BFGS iteration
    ([out, in] x [in, in]; a 1x1 conv [out, in, 1, 1] solves as [out, in])"""
    out_f, in_f = shape[0], math.prod(shape[1:])
    return out_f * in_f * in_f * iters


def fusion_plan(shapes, iters, world):
    """Which rank solves which weight of one fusion stage: shapes {name: weight shape} of the weights the stage solves ->
    plan[r] = sorted names rank r owns.  Longest-processing-time-first greedy on solve_cost (ties broken by name, each
    job to the least-loaded rank, ties to the lowest rank): the most loaded rank carries at most 4/3 of the optimum.  The
    plan depends on names, shapes and `iters` only, so every rank computes the same one before any GPU work."""
    load = [0] * world
    plan = [[] for _ in range(world)]
    for name in sorted(shapes, key=lambda n: (-solve_cost(shapes[n], iters), n)):
        r = min(range(world), key=lambda i: (load[i], i))
        load[r] += solve_cost(shapes[name], iters)
        plan[r].append(name)
    return [sorted(p_) for p_ in plan]


def _sharded(stage, shapes, iters, rank, world, device, args, kw):
    """Runs `stage(*args, **kw)` on this rank's share of `shapes` (fusion_plan) and exchanges the solved weights: every rank
    returns all of them (on the host).  `device`: the device the stage runs on.  A stage that raises on any rank raises on every rank (the failing rank re-raises its own error)
    before the exchange, so no rank is left waiting in a collective."""
    from mos_b200 import dp
    plan = fusion_plan(shapes, iters, world)
    err, owned = None, {}
    try:
        owned = stage(*args, solve_names=plan[rank], **kw)
    except Exception as exc:                  # reported to the other ranks first, then re-raised below
        err = exc
    if not dp.all_ranks_ok(err is None, device):
        if err is not None:
            raise err
        raise RuntimeError(f'{stage.__name__} failed on another rank')
    return {n: w.cpu() for n, w in dp.broadcast_owned(owned, plan, shapes, device).items()}


def compose_concepts(concept_cfg, optimize_textenc_iters, optimize_unet_iters, pretrained_model_path, save_path, suffix,
                     device='cuda', tokenizer=None, log=print):
    """gradient_fusion.py:750-813 on the GPU path.  `pretrained_model_path`: diffusers-layout directory (unet/,
    text_encoder/, tokenizer/[, vae/, scheduler/]); the fused UNet / text encoder and new_concept_cfg.json are written to
    `{save_path}/combined_model_{suffix}` together with the tokenizer that carries the added `<new{k}>` tokens, and the
    base model's vae/ and scheduler/ folders, which the fusion does not change, are copied there byte for byte when they
    exist: the directory loads as a whole pipeline (EDLoRAPipeline.from_pretrained, regionally_controlable_sampling.py).
    With torch.distributed initialised, the layer solves of every stage are sharded over the ranks (fusion_plan): each rank
    replays the recording, solves its own layers and receives the others' (_sharded); the fused model is the one of a
    single process, bit for bit.  Only rank 0 writes it, and every rank returns once it is written."""
    import os
    import torch.distributed as dist
    from mixofshow.pipelines.pipeline_edlora import bind_concept_prompt
    from mixofshow.utils import model_io
    world = dist.get_world_size() if dist.is_initialized() else 1
    rank = dist.get_rank() if world > 1 else 0

    def run(stage, shapes, iters, *args, **kw):
        if world == 1:
            return stage(*args, **kw)
        return _sharded(stage, shapes, iters, rank, world, device, args, kw)
    log('------Step 1: load stable diffusion checkpoint------')
    unet = model_io.load_unet(pretrained_model_path)
    text_encoder = model_io.load_text_encoder(pretrained_model_path, device=device)
    if tokenizer is None:
        from transformers import CLIPTokenizer
        tokenizer = CLIPTokenizer.from_pretrained(pretrained_model_path, subfolder='tokenizer')
    log('------Step 2: load new concepts checkpoints------')
    embedding_list, text_encoder_list, unet_crosskv_list, unet_spatial_attn_list, concept_list = \
        parse_new_concepts(concept_cfg)
    if any(item is not None for item in embedding_list):
        log('------Step 3: merge token embedding------')
        _, new_concept_cfg = merge_new_concepts_(embedding_list, concept_list, tokenizer, text_encoder)
    else:
        new_concept_cfg = {}

    def prompts_of(concept):                                  # 32 layer-bound prompts (:515-520, :381-385)
        return bind_concept_prompt([TEMPLATE_SIMPLE.format(concept['concept_name']), concept['concept_name']],
                                   new_concept_cfg)

    if any(item is not None for item in text_encoder_list):
        log('------Step 4: merge text encoder------')
        ids = [[torch.tensor(_unpadded_ids(p_, tokenizer)) for p_ in prompts_of(c)] for c in concept_list]
        sd = text_encoder.state_dict()
        shapes = {n: tuple(sd[n].shape) for n in lora_weight_names(text_encoder_list)}
        new_w = run(merge_text_encoder, shapes, optimize_textenc_iters, sd, text_encoder_list,
                    [c['text_encoder_alpha'] for c in concept_list], ids, optimize_textenc_iters, device=device)
        sd.update(new_w)
        text_encoder.load_state_dict(sd)
    if any(item is not None for item in unet_crosskv_list):
        log('------Step 5: merge kv of cross-attention in unet------')
        feats = []
        for c in concept_list:
            cp = prompts_of(c)
            n = len(cp) // NUM_CROSS_ATTENTION_LAYERS
            feats.append({i: get_text_feature([cp[j * NUM_CROSS_ATTENTION_LAYERS + i] for j in range(n)], tokenizer,
                                              text_encoder, device).cpu() for i in range(NUM_CROSS_ATTENTION_LAYERS)})
        sd = unet.state_dict()
        kv_names = cross_kv_layer_names(unet)
        shapes = {n: tuple(sd[n].shape) for _, n in kv_names}
        new_w = run(merge_kv_in_cross_attention, shapes, optimize_textenc_iters, sd, kv_names, feats, unet_crosskv_list,
                    [c['unet_alpha'] for c in concept_list], optimize_textenc_iters, device=device)
        sd.update(new_w)
        unet.load_state_dict(sd)
    if any(item is not None for item in unet_spatial_attn_list):
        log('------Step 6: merge spatial attention (q in cross-attention, qkv in self-attention) in unet------')
        embeds = [get_text_feature(bind_concept_prompt([TEMPLATE_SIMPLE.format(c['concept_name'])], new_concept_cfg),
                                   tokenizer, text_encoder, device, return_type='full_embedding').unsqueeze(0).cpu()
                  for c in concept_list]
        cfg = unet.config
        sd = unet.state_dict()
        shapes = {n: tuple(sd[n].shape) for n in lora_weight_names(unet_spatial_attn_list)}
        new_w = run(merge_spatial_attention, shapes, optimize_unet_iters, sd, unet_spatial_attn_list,
                    [c['unet_alpha'] for c in concept_list], embeds, optimize_unet_iters, device=device,
                    block_out=tuple(cfg.block_out_channels), layers=cfg.layers_per_block)
        sd.update(new_w)
        unet.load_state_dict(sd)
    out_dir = os.path.join(save_path, f'combined_model_{suffix}')
    if rank == 0:
        model_io.save_combined_model(out_dir, unet, text_encoder, new_concept_cfg, tokenizer=tokenizer,
                                     base_model=pretrained_model_path)
    if world > 1:
        dist.barrier()
    return out_dir, new_concept_cfg


def parse_args(argv=None):
    import argparse
    parser = argparse.ArgumentParser('', add_help=False)
    parser.add_argument('--concept_cfg', help='json file for multi-concept', required=True, type=str)
    parser.add_argument('--save_path', help='folder name to save optimized weights', required=True, type=str)
    parser.add_argument('--suffix', help='suffix name', default='base', type=str)
    parser.add_argument('--pretrained_models', required=True, type=str)
    parser.add_argument('--optimize_unet_iters', default=50, type=int)
    parser.add_argument('--optimize_textenc_iters', default=500, type=int)
    return parser.parse_args(argv)


def main(argv=None):
    """`python gradient_fusion.py ...`, or under torchrun with the layer solves sharded across the ranks
    (init_distributed, compose_concepts); only rank 0 logs."""
    import torch.distributed as dist
    args = parse_args(argv)
    rank, world, device = init_distributed()
    try:
        if rank == 0:
            os.makedirs(args.save_path, exist_ok=True)
        return compose_concepts(args.concept_cfg, args.optimize_textenc_iters, args.optimize_unet_iters,
                                args.pretrained_models, args.save_path, args.suffix, device=device,
                                log=print if rank == 0 else (lambda *a, **k: None))
    finally:
        if world > 1:
            dist.destroy_process_group()

if __name__ == '__main__':
    main()
