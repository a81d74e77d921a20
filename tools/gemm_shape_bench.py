"""Per-shape timing of the wgmma GEMM / implicit-GEMM conv launches of one denoise step (the bench.py workload).

Records every ops.gemm call of one eager step on the real engine buffers, groups the calls by their full argument set,
and replays each group back to back between CUDA events (same arguments, so the same kernel parameters).  Per shape it
prints us per launch, achieved TFLOP/s (2*M*N*K), and the tensor-rate bound: ceil(items / SMs) * (k blocks per item)
* 640 cycles (one 128x160x64 k block at 4096 dense 16-bit FLOP/clk/SM) at the card's maximum SM clock.  With the
in-kernel timeline (mos_debug_set_timeline, 16 stamps per CTA, listed in csrc/gemm.cu) it prints the phase split of
the first work item of the first 8 CTAs (medians over the CTAs that stamped both ends of a phase):
  tma1   launch -> first k block landed            main   -> accumulators ready
  ops    -> epilogue operands in shared memory     rdy    -> epi_ready passed (residual landed)
  stage  -> staging tile written                   wake   -> the producer observed epi_full
  issue  -> TMA stores issued                      drain  -> the stores have read the staging tile
  epi    accumulators ready -> tile written (ops + rdy + stage + wake + issue + drain)
and `epi2`, the same epilogue phase of the second work item in CTAs that run several.  `cyc/kb` is the mainloop per k
block in SM cycles at the bound clock (640 at the tensor rate), and `opMB` the operand bytes the launch moves from L2
into shared memory (items x k blocks x stage bytes).  A CTA with several tiles writes
a tile out only after issuing the next tile's k blocks, so there `epi` includes that wait.  On the copy-out path (no
TMA stores) the consumers write the tile and `wake`, `issue` and `drain` are empty.

The replay calls ops.gemm, which encodes the tensor maps on the host at every launch: a launch shorter than that host
work is timed at the host's rate, so compare short launches against the bound with the timeline's phases.

    python tools/gemm_shape_bench.py [--reps 50] [--max-ctas N] [--out DIR]

--max-ctas caps the persistent grid (MOS_GEMM_MAX_CTAS): a k block that gets faster when fewer SMs run is contending
for a resource the SMs share (L2 bandwidth), not bound inside the SM.
"""
import argparse
import ctypes
import json
import math
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, 'mix-of-show_b200')):
    sys.path.insert(0, p)

BM, BN, BK = 128, 160, 64
CYCLES_PER_KBLOCK = BM * BN * BK * 2 // 4096     # 640
A_STAGE_BYTES, B_STAGE_BYTES, LORA_STAGE_BYTES = BM * BK * 2, BN * BK * 2, 16 * BK * 2


def conv_m_tiles(B, H, Wd):
    """Row tiles of an implicit-GEMM conv launch: the TW x TH x TB patch choice of mos_gemm_bf16 (csrc/gemm.cu)."""
    TW = 1
    while TW * 2 <= 128 and Wd % (TW * 2) == 0:
        TW *= 2
    best_th, best_eff, TH = 1, -1.0, 1
    while TH * TW <= 128:
        TB = 128 // (TW * TH)
        if not (TB > 4 and TH * 2 * TW <= 128):
            eff = (H / (math.ceil(H / TH) * TH)) * (B / (math.ceil(B / TB) * TB))
            if eff > best_eff + 1e-9:
                best_eff, best_th = eff, TH
        TH *= 2
    TB = 128 // (TW * best_th)
    return (Wd // TW) * math.ceil(H / best_th) * math.ceil(B / TB)


def describe(A, W, kw):
    """(M, N, K, flops, items, k blocks per item, label) of one ops.gemm call."""
    conv = kw.get('conv')
    N, K = W.shape[0], W.shape[1]
    if conv is not None:
        B, H, Wd, C = conv
        M, K = B * H * Wd, C
        m_tiles, kb = conv_m_tiles(B, H, Wd), 9 * C // BK
    else:
        M = kw.get('M') or A.shape[0]
        m_tiles, kb = math.ceil(M / BM), K // BK
    splits = kw.get('splits') or 1
    kind = []
    if conv is not None:
        kind.append('conv')
    if kw.get('lora_down') is not None:
        kind.append('lora')
    if kw.get('geglu'):
        kind.append('geglu')
    if kw.get('heads') is not None:
        kind.append('heads')
    if kw.get('out_f32'):
        kind.append('f32' + ('+acc' if kw.get('accumulate') else ''))
    if kw.get('residual') is not None:
        kind.append('res')
    if splits > 1:
        kind.append(f'splitk{splits}' + ('+fin' if kw.get('counters') is not None else ''))
    flops = 2.0 * M * N * (9 * K if conv is not None else K)
    return M, N, K, flops, (N // BN) * m_tiles * splits, math.ceil(kb / splits), ','.join(kind) or 'plain'


def arg_key(A, W, out, kw):
    def k(v):
        if hasattr(v, 'data_ptr'):
            return ('T', v.data_ptr(), tuple(v.shape), tuple(v.stride()), str(v.dtype))
        if isinstance(v, dict):
            return tuple(sorted((a, k(b)) for a, b in v.items()))
        if isinstance(v, (list, tuple)):
            return tuple(k(x) for x in v)
        return v
    return (k(A), k(W), k(out), tuple(sorted((a, k(b)) for a, b in kw.items())))


def card_info():
    """Name, power limit and SM clocks (queries only), read in the same process as the measurement."""
    q = 'name,power.limit,clocks.sm,clocks.max.sm'
    try:
        r = subprocess.run(['nvidia-smi', f'--query-gpu={q}', '--format=csv,noheader,nounits'],
                           capture_output=True, text=True, timeout=30)
        vals = [v.strip() for v in r.stdout.strip().splitlines()[0].split(',')]
        return dict(zip(['name', 'power_limit_w', 'sm_mhz', 'max_sm_mhz'], vals))
    except (OSError, IndexError, subprocess.SubprocessError) as e:
        return {'error': repr(e)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=50, help='timed launches per shape (after 5 warm-up launches)')
    ap.add_argument('--out', default=None, help='also write the table as DIR/gemm_shapes.json')
    ap.add_argument('--max-ctas', type=int, default=0, help='cap the persistent grid at N CTAs (MOS_GEMM_MAX_CTAS)')
    args = ap.parse_args()
    if args.max_ctas > 0:
        os.environ['MOS_GEMM_MAX_CTAS'] = str(args.max_ctas)     # read once, at the first launch
    import torch
    assert torch.cuda.is_available(), 'gemm_shape_bench.py needs a GPU'
    import bench
    from mos_b200 import _lib, ops

    dev = torch.device('cuda', 0)
    sd, lora, lat, ehs, cfg = bench.build_workload(False, 1)
    pipe = bench.build_pipeline(sd, lora, cfg, dev)
    unet = pipe.unet
    unet.act_dtype = torch.float16
    B, H, W = 2, lat.shape[2], lat.shape[3]
    eng = unet.session(B, H, W, dev, ehs.to(dev)).eng
    eng.in_latents.copy_(torch.cat([lat, lat]).to(dev))
    eng.in_t.fill_(981.0)
    eng.run()
    eng.run()
    torch.cuda.synchronize()

    calls = []
    orig = ops.gemm

    def recording(A, W, out=None, **kw):
        calls.append((A, W, out, kw))
        return orig(A, W, out, **kw)

    ops.gemm = recording
    try:
        eng._run()
        torch.cuda.synchronize()
    finally:
        ops.gemm = orig

    groups = {}
    for c in calls:
        groups.setdefault(arg_key(*c), []).append(c)
    info = card_info()
    n_sm = torch.cuda.get_device_properties(0).multi_processor_count
    try:
        clk_ghz = float(info['max_sm_mhz']) / 1e3
    except (KeyError, ValueError):          # not reported (e.g. '[N/A]'): the H100 SXM maximum
        clk_ghz = 1.98

    lib = _lib.lib()
    TL_SLOTS = 16
    tl = torch.zeros(8 * TL_SLOTS, dtype=torch.int64, device=dev)
    rows = []
    for calls_g in groups.values():
        A, W, out, kw = calls_g[0]
        M, N, K, flops, items, kbi, label = describe(A, W, kw)
        for _ in range(5):
            orig(A, W, out, **kw)
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(args.reps):
            orig(A, W, out, **kw)
        e1.record()
        torch.cuda.synchronize()
        us = 1e3 * e0.elapsed_time(e1) / args.reps
        # one launch with the timeline registered (stamps of the first work item, first 8 CTAs)
        tl.zero_()
        torch.cuda.synchronize()
        _lib.check(lib.mos_debug_set_timeline(ctypes.c_void_p(tl.data_ptr())), 'mos_debug_set_timeline')
        try:
            orig(A, W, out, **kw)
            torch.cuda.synchronize()
        finally:
            _lib.check(lib.mos_debug_set_timeline(None), 'mos_debug_set_timeline')
        st = tl.view(8, TL_SLOTS).cpu().tolist()
        ncta = min(8, items)

        def med(a, b):
            v = sorted((s[b] - s[a]) / 1e3 for s in st[:ncta] if s[a] and s[b])
            return v[len(v) // 2] if v else float('nan')

        bound_us = math.ceil(items / n_sm) * kbi * CYCLES_PER_KBLOCK / (clk_ghz * 1e3)
        stage = A_STAGE_BYTES + B_STAGE_BYTES + (LORA_STAGE_BYTES if kw.get('lora_down') is not None else 0)
        main_us = med(3, 4)
        rows.append(dict(cycles_per_kb=main_us * clk_ghz * 1e3 / kbi, operand_mb=items * kbi * stage / 1e6,
                         M=M, N=N, K=K, kind=label, count=len(calls_g), items=items, kb_per_item=kbi, us=us,
                         tflops=flops / (us * 1e-6) / 1e12, bound_us=bound_us,
                         first_tma_us=med(1, 3), mainloop_us=main_us, epilogue_us=med(4, 5),
                         ops_us=med(4, 6), ready_us=med(6, 7), stage_us=med(7, 8), wake_us=med(8, 9),
                         issue_us=med(9, 10), drain_us=med(10, 5), epilogue2_us=med(11, 15)))
    rows.sort(key=lambda r: -r['us'] * r['count'])
    print(f"card: {info}  SMs {n_sm}  grid cap {args.max_ctas or n_sm}  bound clock {clk_ghz:.3f} GHz  "
          f"launches/step {len(calls)}")
    hdr = (f"{'M':>6} {'N':>5} {'K':>5} {'kind':<18} {'n':>3} {'items':>5} {'kb':>4} {'us':>8} {'TF/s':>6} "
           f"{'bound':>7} {'tma1':>6} {'main':>7} {'epi':>6} {'ops':>6} {'rdy':>6} {'stage':>6} {'wake':>6} "
           f"{'issue':>6} {'drain':>6} {'epi2':>6} {'cyc/kb':>7} {'opMB':>7}")
    print(hdr)
    for r in rows:
        print(f"{r['M']:>6} {r['N']:>5} {r['K']:>5} {r['kind']:<18} {r['count']:>3} {r['items']:>5} "
              f"{r['kb_per_item']:>4} {r['us']:>8.2f} {r['tflops']:>6.1f} {r['bound_us']:>7.2f} "
              f"{r['first_tma_us']:>6.2f} {r['mainloop_us']:>7.2f} {r['epilogue_us']:>6.2f} {r['ops_us']:>6.2f} "
              f"{r['ready_us']:>6.2f} {r['stage_us']:>6.2f} {r['wake_us']:>6.2f} {r['issue_us']:>6.2f} "
              f"{r['drain_us']:>6.2f} {r['epilogue2_us']:>6.2f} {r['cycles_per_kb']:>7.0f} {r['operand_mb']:>7.1f}")
    tot = sum(r['us'] * r['count'] for r in rows)
    bnd = sum(r['bound_us'] * r['count'] for r in rows)
    opb = sum(r['operand_mb'] * r['count'] for r in rows)
    print(f"step total: {tot / 1e3:.3f} ms of back-to-back launches, tensor-rate bound {bnd / 1e3:.3f} ms, "
          f"operand bytes {opb / 1e3:.2f} GB")
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, 'gemm_shapes.json'), 'w') as f:
            json.dump({'card': info, 'max_ctas': args.max_ctas or n_sm, 'rows': rows, 'total_ms': tot / 1e3,
                       'bound_ms': bnd / 1e3, 'operand_gb': opb / 1e3}, f, indent=1)


if __name__ == '__main__':
    main()
