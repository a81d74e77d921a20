// lbfgs.cu — native driver of the per-layer least-squares solves of gradient fusion (gradient_fusion.py:38-96):
// ONE torch.optim.LBFGS.step(closure) with line_search_fn='strong_wolfe', history 25, on the Gram-form objective
//     f(D) = s <D, D G - 2 R> + f0,   grad = 2 s (D G - R),   D = W - W0
// (see fusion.cu for the derivation).  The reference drives this loop from Python with one closure per evaluation that
// streams GBs of features from host memory; here the whole loop is host C++ inside the library: every vector operation is
// one of the mos_vec_* / mos_lbfgs_direction / mos_dgemm_mixed / mos_ls_grad_loss launches (same kernels, same order and
// therefore the same bits as the Python driver kept in mix-of-show_b200/gradient_fusion.py::lbfgs_minimize), the handful of
// scalars a line search needs come back through a pinned buffer, and mos_lbfgs_solve_batch runs the independent layers of a
// fusion stage on several host threads x CUDA streams (no interpreter lock).
#include <math.h>

#include <algorithm>
#include <atomic>
#include <cmath>
#include <thread>
#include <vector>

#include "common.h"

namespace {

struct Pt {        // a point of the line search: step, value, gradient buffer (slot of the ring, -1 = caller's g), <grad, d>
  double t, f;
  int g;
  double gtd;
};

// Minimiser of the cubic through (x1,f1,g1), (x2,f2,g2), clipped to the bounds (Nocedal & Wright eq. 3.59), as
// torch.optim.lbfgs._cubic_interpolate
double cubic_min(double x1, double f1, double g1, double x2, double f2, double g2, bool has_bounds, double blo, double bhi) {
  double lo, hi;
  if (has_bounds) {
    lo = blo;
    hi = bhi;
  } else if (x1 <= x2) {
    lo = x1;
    hi = x2;
  } else {
    lo = x2;
    hi = x1;
  }
  const double d1 = g1 + g2 - 3.0 * (f1 - f2) / (x1 - x2);
  const double disc = d1 * d1 - g1 * g2;
  if (disc < 0) return 0.5 * (lo + hi);
  const double d2 = sqrt(disc);
  double pos;
  if (x1 <= x2) pos = x2 - (x2 - x1) * ((g2 + d2 - d1) / (g2 - g1 + 2.0 * d2));
  else pos = x1 - (x1 - x2) * ((g1 + d2 - d1) / (g1 - g2 + 2.0 * d2));
  return std::min(std::max(pos, lo), hi);
}

constexpr int MAX_LS = 25;
constexpr int RING = MAX_LS + 2;

struct Solver {
  const mos_lbfgs_problem& P;
  cudaStream_t st;
  void* stv;
  long long n;
  int H;
  // device
  float *x, *g, *prev_g, *d, *xt;
  float* ring[RING];
  // curvature pairs in two rings of H + 1 slots (the extra slot holds the candidate pair of the current iteration): logical
  // pair i (0 = oldest) lives in physical slot (head + i) % slots
  float *S_ring, *Y_ring;
  int slots, head = 0, k = 0;
  std::vector<double> rho_phys;
  double *Y64, *loss64, *scratch64, *work, *d_rho;
  float *scal, *scratch, *partial, *gtd_dev, *d_hdiag;
  int* d_head;
  struct Stage {            // pinned: values uploaded before a direction
    int head;
    float hdiag;
    double rho[64];
  }* stage = nullptr;
  cudaGraph_t graph = nullptr;
  cudaGraphExec_t graph_exec = nullptr;
  // pinned host scalars
  double* h_d;
  float* h_f;
  double best_loss = INFINITY;
  int evals = 0;
  int rc = MOS_OK;

  Solver(const mos_lbfgs_problem& p, cudaStream_t s) : P(p), st(s), stv(reinterpret_cast<void*>(s)) {
    n = (long long)p.out_f * p.in_f;
    H = p.history > 0 ? p.history : 25;
    slots = H + 1;
    rho_phys.assign(slots, 0.0);
  }
  ~Solver() {
    if (graph_exec) cudaGraphExecDestroy(graph_exec);
    if (graph) cudaGraphDestroy(graph);
  }

  static size_t align_up(size_t v) { return (v + 255) & ~size_t(255); }
  static size_t workspace_bytes(long long n, int H) {
    size_t b = 0;
    b += align_up(sizeof(float) * n) * (5 + RING);
    b += 2 * align_up(sizeof(float) * n * ((size_t)H + 1));  // S / Y rings (H pairs + the candidate of the current iteration)
    b += align_up(sizeof(double) * n);                       // Y64
    b += align_up(sizeof(double) * (1 + 256 + 64 + 64));     // loss64, scratch64, work, rho
    b += align_up(sizeof(float) * (8 + 256 + 260 + 4));      // scal, scratch, partial, gtd
    return b;
  }
  void carve(void* ws) {
    uint8_t* p = reinterpret_cast<uint8_t*>(ws);
    auto takef = [&](long long cnt) {
      float* r = reinterpret_cast<float*>(p);
      p += align_up(sizeof(float) * cnt);
      return r;
    };
    x = takef(n), g = takef(n), prev_g = takef(n), d = takef(n), xt = takef(n);
    for (int i = 0; i < RING; ++i) ring[i] = takef(n);
    S_ring = takef(n * (long long)slots);
    Y_ring = takef(n * (long long)slots);
    Y64 = reinterpret_cast<double*>(p);
    p += align_up(sizeof(double) * n);
    loss64 = reinterpret_cast<double*>(p);
    scratch64 = loss64 + 1;
    work = scratch64 + 256;
    d_rho = work + 64;
    p += align_up(sizeof(double) * (1 + 256 + 64 + 64));
    scal = reinterpret_cast<float*>(p);
    scratch = scal + 8;
    partial = scratch + 256;
    gtd_dev = partial + 260;
    d_hdiag = scal + 4;
    d_head = reinterpret_cast<int*>(scal + 5);
  }

#define CK(call)              \
  do {                        \
    if (rc == MOS_OK) {       \
      int r_ = (call);        \
      if (r_ != MOS_OK) rc = r_; \
    }                         \
  } while (0)
#define CKC(call)                                           \
  do {                                                      \
    if (rc == MOS_OK && (call) != cudaSuccess) rc = MOS_ECUDA; \
  } while (0)

  void sync() { CKC(cudaStreamSynchronize(st)); }
  // n_f floats from scal[0..] and optionally the loss double, one synchronisation
  void fetch(int n_f, bool with_loss) {
    if (n_f > 0) CKC(cudaMemcpyAsync(h_f, scal, sizeof(float) * n_f, cudaMemcpyDeviceToHost, st));
    if (with_loss) CKC(cudaMemcpyAsync(h_d, loss64, sizeof(double), cudaMemcpyDeviceToHost, st));
    sync();
  }
  void copy(float* dst, const float* src) { CKC(cudaMemcpyAsync(dst, src, sizeof(float) * n, cudaMemcpyDeviceToDevice, st)); }
  void axpby(float* y, const float* xx, double a, double b) { CK(mos_vec_axpby(y, xx, (float)a, (float)b, n, stv)); }
  double absmax(const float* a, double scale) {
    CK(mos_vec_absmax(a, n, (float)scale, scal, scratch, stv));
    fetch(1, false);
    return (double)h_f[0];
  }

  // closure at `pt` (gradient into `grad`) + <grad, dvec> (dvec may be NULL): loss, gtd with ONE synchronisation
  void closure(const float* pt, float* grad, const float* dvec, double& loss, double& gtd) {
    CK(mos_dgemm_mixed(pt, P.G, Y64, P.out_f, P.in_f, P.in_f, stv));
    CK(mos_ls_grad_loss(pt, Y64, P.R, n, P.s, P.f0, grad, loss64, scratch64, stv));
    if (dvec != nullptr) CK(mos_vec_dot(grad, dvec, n, scal, scratch, stv));
    fetch(dvec != nullptr ? 1 : 0, true);
    loss = h_d[0];
    gtd = dvec != nullptr ? (double)h_f[0] : 0.0;
    ++evals;
    // the reference keeps the best iterate of all evaluations (:72-74); a non-finite loss never qualifies, so a solve whose
    // G or R holds NaN / Inf ends with best_loss = INFINITY and P.best_D unwritten (solve_one then fails)
    if (std::isfinite(loss) && loss < best_loss) {
      best_loss = loss;
      copy(P.best_D, pt);
    }
  }

  // strong-Wolfe line search (bracketing + zoom with cubic interpolation) of torch.optim.LBFGS
  void strong_wolfe(double t, double f, double gtd, double& f_out, int& g_out, double& t_out, int& ls_evals) {
    const double c1 = 1e-4, c2 = 0.9, tol_change = 1e-9;
    const double d_norm = absmax(d, 1.0);
    int next_slot = 0;
    auto phi = [&](double step) {
      Pt r;
      r.t = step;
      r.g = next_slot++;
      copy(xt, x);
      axpby(xt, d, step, 1.0);
      closure(xt, ring[r.g], d, r.f, r.gtd);
      return r;
    };
    Pt cur = phi(t);
    ls_evals = 1;
    Pt prev = {0.0, f, -1, gtd};
    bool done = false;
    int it = 0;
    Pt br[2];
    int nbr = 0;
    while (it < MAX_LS && rc == MOS_OK) {
      if (cur.f > f + c1 * cur.t * gtd || (it > 1 && cur.f >= prev.f)) {
        br[0] = prev, br[1] = cur, nbr = 2;
        break;
      }
      if (fabs(cur.gtd) <= -c2 * gtd) {
        br[0] = cur, nbr = 1;
        done = true;
        break;
      }
      if (cur.gtd >= 0) {
        br[0] = prev, br[1] = cur, nbr = 2;
        break;
      }
      const double lo = cur.t + 0.01 * (cur.t - prev.t), hi = cur.t * 10.0;
      const double t_next = cubic_min(prev.t, prev.f, prev.gtd, cur.t, cur.f, cur.gtd, true, lo, hi);
      prev = cur;
      cur = phi(t_next);
      ++ls_evals;
      ++it;
    }
    if (nbr == 0) {            // it == max_ls
      br[0] = {0.0, f, -1, gtd};
      br[1] = cur;
      nbr = 2;
    }
    bool stalled = false;
    int low = 0, high = 1;
    if (nbr == 2) {
      if (br[0].f <= br[1].f) low = 0, high = 1;
      else low = 1, high = 0;
    }
    while (!done && it < MAX_LS && rc == MOS_OK) {
      if (fabs(br[1].t - br[0].t) * d_norm < tol_change) break;
      double tt = cubic_min(br[0].t, br[0].f, br[0].gtd, br[1].t, br[1].f, br[1].gtd, false, 0, 0);
      const double tmax = std::max(br[0].t, br[1].t), tmin = std::min(br[0].t, br[1].t);
      const double eps = 0.1 * (tmax - tmin);
      if (std::min(tmax - tt, tt - tmin) < eps) {
        if (stalled || tt >= tmax || tt <= tmin) {
          tt = (fabs(tt - tmax) < fabs(tt - tmin)) ? tmax - eps : tmin + eps;
          stalled = false;
        } else {
          stalled = true;
        }
      } else {
        stalled = false;
      }
      cur = phi(tt);
      ++ls_evals;
      ++it;
      if (cur.f > f + c1 * cur.t * gtd || cur.f >= br[low].f) {
        br[high] = cur;
        if (br[0].f <= br[1].f) low = 0, high = 1;
        else low = 1, high = 0;
      } else {
        if (fabs(cur.gtd) <= -c2 * gtd) done = true;
        else if (cur.gtd * (br[high].t - br[low].t) >= 0) br[high] = br[low];
        br[low] = cur;
      }
    }
    const Pt& sel = (nbr == 1) ? br[0] : br[low];
    f_out = sel.f, g_out = sel.g, t_out = sel.t;
  }

  void run() {
    const double tol_grad = 1e-16, tol_change = 1e-16, lr = 1.0;
    const int max_iter = P.max_iter;
    const int max_eval = max_iter * 5 / 4;
    CKC(cudaMemsetAsync(x, 0, sizeof(float) * n, st));                    // D0 = 0
    CKC(cudaMemsetAsync(partial, 0, sizeof(float) * 264, st));           // partial sums + block counter + <g, d>
    double loss, unused;
    closure(x, g, nullptr, loss, unused);
    int total_evals = 1;
    if (absmax(g, 1.0) <= tol_grad) return;
    double h_diag = 1.0, t = 0.0, prev_loss = 0.0;
    int n_iter = 0;
    while (n_iter < max_iter && rc == MOS_OK) {
      ++n_iter;
      double gtd;
      if (n_iter == 1) {
        copy(d, g);
        axpby(d, g, -1.0, 0.0);                                          // d = -g
      } else {
        const int cand = (head + k) % slots;                             // physical slot of the candidate pair
        float* y = Y_ring + (long long)cand * n;
        float* s = S_ring + (long long)cand * n;
        copy(y, g);
        axpby(y, prev_g, -1.0, 1.0);                                     // y = g - prev_g
        axpby(s, d, t, 0.0);                                             // s = t d
        CK(mos_vec_dot(y, s, n, scal, scratch, stv));
        CK(mos_vec_dot(y, y, n, scal + 1, scratch, stv));
        fetch(2, false);
        const double ys = (double)h_f[0], yy = (double)h_f[1];
        if (ys > 1e-10) {
          if (k == H) head = (head + 1) % slots;                          // history full: the oldest pair leaves
          else ++k;
          rho_phys[cand] = 1.0 / ys;
          h_diag = ys / yy;
        }
        stage->head = head;
        stage->hdiag = (float)h_diag;
        for (int i = 0; i < slots; ++i) stage->rho[i] = rho_phys[i];
        CKC(cudaMemcpyAsync(d_hdiag, &stage->hdiag, sizeof(float), cudaMemcpyHostToDevice, st));
        CKC(cudaMemcpyAsync(d_head, &stage->head, sizeof(int), cudaMemcpyHostToDevice, st));
        CKC(cudaMemcpyAsync(d_rho, stage->rho, sizeof(double) * slots, cudaMemcpyHostToDevice, st));
        if (k == H && rc == MOS_OK) {
          // full history: the 2H + 1 launches of the direction have the same parameters on every iteration -> one graph launch
          if (graph_exec == nullptr) {
            CKC(cudaStreamBeginCapture(st, cudaStreamCaptureModeThreadLocal));
            CK(mos_lbfgs_direction_ring(S_ring, Y_ring, slots, d_head, d_rho, d_hdiag, k, g, n, d, work, partial, gtd_dev, stv));
            cudaGraph_t gr = nullptr;
            if (cudaStreamEndCapture(st, &gr) != cudaSuccess || gr == nullptr) rc = rc == MOS_OK ? MOS_ECUDA : rc;
            graph = gr;
            if (rc == MOS_OK) CKC(cudaGraphInstantiate(&graph_exec, graph, 0));
          }
          if (rc == MOS_OK) CKC(cudaGraphLaunch(graph_exec, st));
        } else {
          CK(mos_lbfgs_direction_ring(S_ring, Y_ring, slots, d_head, d_rho, d_hdiag, k, g, n, d, work, partial, gtd_dev, stv));
        }
      }
      copy(prev_g, g);
      prev_loss = loss;
      if (n_iter == 1) {
        CK(mos_vec_asum(g, n, scal, scratch, stv));                      // |g|_1
        CK(mos_vec_dot(g, d, n, scal + 1, scratch, stv));
        fetch(2, false);
        t = std::min(1.0, 1.0 / (double)h_f[0]) * lr;
        gtd = (double)h_f[1];
      } else {
        t = lr;
        CKC(cudaMemcpyAsync(h_f, gtd_dev, sizeof(float), cudaMemcpyDeviceToHost, st));
        sync();
        gtd = (double)h_f[0];
      }
      if (gtd > -tol_change) break;
      int g_sel, ls_evals;
      double f_sel, t_sel;
      strong_wolfe(t, loss, gtd, f_sel, g_sel, t_sel, ls_evals);
      loss = f_sel;
      t = t_sel;
      if (g_sel >= 0) copy(g, ring[g_sel]);
      axpby(x, d, t, 1.0);
      total_evals += ls_evals;
      if (n_iter == max_iter || total_evals >= max_eval) break;
      CK(mos_vec_absmax(g, n, 1.0f, scal, scratch, stv));
      CK(mos_vec_absmax(d, n, (float)t, scal + 1, scratch, stv));
      fetch(2, false);
      if ((double)h_f[0] <= tol_grad || (double)h_f[1] <= tol_change || fabs(loss - prev_loss) < tol_change) break;
    }
  }
};

int solve_one(const mos_lbfgs_problem& p, void* workspace, cudaStream_t st) {
  Solver s(p, st);
  s.carve(workspace);
  void* pinned = nullptr;
  if (cudaHostAlloc(&pinned, 64 + sizeof(Solver::Stage), cudaHostAllocDefault) != cudaSuccess) return MOS_ECUDA;
  s.h_d = reinterpret_cast<double*>(pinned);
  s.h_f = reinterpret_cast<float*>(reinterpret_cast<uint8_t*>(pinned) + 16);
  s.stage = reinterpret_cast<Solver::Stage*>(reinterpret_cast<uint8_t*>(pinned) + 64);
  s.run();
  cudaStreamSynchronize(st);
  cudaFreeHost(pinned);
  if (p.best_loss != nullptr) *p.best_loss = s.best_loss;
  if (p.n_evals != nullptr) *p.n_evals = s.evals;
  if (s.rc == MOS_OK && !std::isfinite(s.best_loss)) return MOS_EINVAL;   // no finite evaluation: best_D is unwritten
  return s.rc;
}

const char* solve_failure(int rc) {
  return rc == MOS_EINVAL ? "no closure evaluation gave a finite loss (G or R holds NaN or Inf); best_D left unwritten"
                          : "CUDA error";
}

bool valid(const mos_lbfgs_problem& p) {
  return p.G && p.R && p.best_D && p.out_f > 0 && p.in_f > 0 && p.max_iter > 0 && p.history >= 0 && p.history <= 63;
}

}  // namespace

extern "C" int64_t mos_lbfgs_workspace_bytes(int32_t out_f, int32_t in_f, int32_t history) {
  return (int64_t)Solver::workspace_bytes((long long)out_f * in_f, history > 0 ? history : 25);
}

extern "C" int mos_lbfgs_solve(const mos_lbfgs_problem* p, void* workspace, void* stream) {
  MOS_CHECK_ARG(p != nullptr && workspace != nullptr && valid(*p), "mos_lbfgs_solve: bad arguments");
  const int rc = solve_one(*p, workspace, reinterpret_cast<cudaStream_t>(stream));
  MOS_CHECK_ARG(rc != MOS_EINVAL, "mos_lbfgs_solve: %s", solve_failure(rc));
  return rc;
}

extern "C" int mos_lbfgs_solve_batch(const mos_lbfgs_problem* probs, int32_t n_probs, int32_t workers) {
  MOS_CHECK_ARG(probs != nullptr && n_probs > 0 && workers > 0, "mos_lbfgs_solve_batch: bad arguments");
  for (int i = 0; i < n_probs; ++i) MOS_CHECK_ARG(valid(probs[i]), "mos_lbfgs_solve_batch: bad problem %d", i);
  int dev = 0;
  MOS_CHECK_CUDA(cudaGetDevice(&dev));
  MOS_CHECK_CUDA(cudaDeviceSynchronize());          // the problems were assembled on the caller's streams
  // largest problems first: the tail of the schedule is then filled with short solves
  std::vector<int> order(n_probs);
  for (int i = 0; i < n_probs; ++i) order[i] = i;
  std::stable_sort(order.begin(), order.end(), [&](int a, int b) {
    return (long long)probs[a].out_f * probs[a].in_f > (long long)probs[b].out_f * probs[b].in_f;
  });
  size_t ws_bytes = 0;
  for (int i = 0; i < n_probs; ++i)
    ws_bytes = std::max(ws_bytes, Solver::workspace_bytes((long long)probs[i].out_f * probs[i].in_f,
                                                          probs[i].history > 0 ? probs[i].history : 25));
  const int nw = std::min<int>(workers, n_probs);
  std::atomic<int> next(0), err(MOS_OK), failed(-1);   // failed: index of the first problem whose solve failed
  auto worker = [&]() {
    if (cudaSetDevice(dev) != cudaSuccess) {
      err = MOS_ECUDA;
      return;
    }
    cudaStream_t st = nullptr;
    void* ws = nullptr;
    if (cudaStreamCreateWithFlags(&st, cudaStreamNonBlocking) != cudaSuccess || cudaMalloc(&ws, ws_bytes) != cudaSuccess) {
      err = MOS_ECUDA;
      if (st) cudaStreamDestroy(st);
      return;
    }
    for (;;) {
      const int j = next.fetch_add(1);
      if (j >= n_probs || err.load() != MOS_OK) break;
      const int rc = solve_one(probs[order[j]], ws, st);
      if (rc != MOS_OK) {
        int none = -1;
        if (failed.compare_exchange_strong(none, order[j])) err = rc;
      }
    }
    cudaStreamSynchronize(st);
    cudaFree(ws);
    cudaStreamDestroy(st);
  };
  std::vector<std::thread> threads;
  for (int i = 0; i < nw; ++i) threads.emplace_back(worker);
  for (auto& t : threads) t.join();
  MOS_CHECK_CUDA(cudaDeviceSynchronize());
  const int rc = err.load();
  if (rc != MOS_OK)
    return ::mos::set_err(rc, "mos_lbfgs_solve_batch: problem %d: %s", failed.load() >= 0 ? failed.load() : -1,
                   failed.load() >= 0 ? solve_failure(rc) : "a worker could not create its stream or workspace");
  return MOS_OK;
}
