#!/usr/bin/env python
"""bench.py — BASELINE.json's metric on BASELINE.json's configs, all five under one clock.

  python bench.py --gpus N --steps K --warmup W            # this repo (sm_90a kernels through the C ABI)
  python bench.py --impl reference --gpus N --steps K ...  # the reference's own CPU kernels on the host cores

ONE JSON line on stdout (rank 0). The headline fields are BASELINE `configs[1]` (workload `c2`); `"configs": {"c1": …, "c3": …,
"c4": …, "c5": …}` carries the other four, each with value / e2e / roofline / cpu_baseline / parity, so every BASELINE config has a
driver-clocked number (`--workload cX` runs one of them alone and prints it as the line).

  c2 (headline) synthetic 1M x 768 float32 unit rows (latent-factor model, generated ON THE DEVICE, seeds fixed), DOT_PRODUCT, Vamana
     graph M=32 efConstruction=100 overflow 1.2 alpha 1.2 with hierarchy (device builder, untimed set-up), GraphSearcher top-10 with
     rerankK = 10 x overquery (default 10). A step = one batch of nq = 10 000 queries searched to completion. Replica per GPU.
  c1 siftsmall 10k x 128 exact L2 (tests/golden/siftsmall): graph search + brute force against the shipped ground truth.
  c3 the c2 data through PQ (M=96, k=256): ADC walk over the FusedPQ records + float32 rerank.
  c4 synthetic 1M x 1536 BQ, Hamming top-100 of 1000 queries; the base RANGE-SHARDED over the N ranks, one NCCL all-gather of the
     per-rank keys + device merge per step (strong scaling).
  c5 GraphIndexBuilder build of 10M x 768 (rows generated on the device) + NVQ encode of every row.

value   : units/s with inputs already resident in HBM, device time from CUDA events on the launching stream
e2e     : the same through the host-pointer C-ABI call (H2D of the inputs and D2H of the results inside the timed region)
roofline: the dominant kernel's algorithmic bytes (or ops) per launch / its launch time, vs MEASURED_PEAKS.json
cpu_baseline / --impl reference: the oracle traversal driver calling the reference's own compiled kernels (oracle/_ref/libjvector.so)
          on the host cores: base rows in NUMA-interleaved memory, a thread sweep, the best thread count reported.
parity  : device results against the oracle at the bench's own scale (ids, keys, sampled scores) — true / false per check.
"""
import argparse
import ctypes as C
import json
import os

# several ranks share one host: keep each rank's BLAS / OpenMP pools to its share of the cores (data generation only)
_world = int(os.environ.get("WORLD_SIZE", "1"))
if _world > 1:
    _share = str(max(1, (os.cpu_count() or 1) // _world))
    for _v in ("OMP_NUM_THREADS", "OPENBLAS_NUM_THREADS", "MKL_NUM_THREADS"):
        os.environ.setdefault(_v, _share)
import subprocess
import sys
import threading
import time
import traceback

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

SEED = 20260922
LATENT = 32      # intrinsic dimensionality of the synthetic embedding model
NOISE = 0.25     # isotropic noise relative to the per-coordinate signal
# NVIDIA's H100 SXM data sheet (700 W card): dense INT8 tensor-core rate and HBM3 bandwidth. Data-sheet figures, not measured.
I8_PEAK_TOPS = 1979.0
HBM_PEAK_GBS = 3350.0
# what the timed paths computed in their last step, written by --dump-outputs: name -> array
DUMP = {}


def log(*a):
    print(*a, file=sys.stderr, flush=True)


def gen_unit_rows_device(torch, seed, n, dim, dist="latent", chunk=262144, device="cuda"):
    """Synthetic float32 unit rows generated ON THE DEVICE (torch is plumbing here: RNG + one small matmul per chunk).
    dist="latent": x = normalise(z A + NOISE * e), z ~ N(0, I_32), A a fixed 32 x dim Gaussian map, e ~ N(0, I_dim): embedding-like
        data with neighbourhood structure, so recall@10 is a meaningful axis.
    dist="iid": i.i.d. N(0,1) rows normalised (SURVEY §8d's first suggestion; graph search on 1M x 768 i.i.d. rows reaches recall@10
        ~ 0.05 for the reference traversal and this one alike — distance concentration — so it is an option, not the headline)."""
    g = torch.Generator(device=device)
    g.manual_seed(seed)
    out = torch.empty((n, dim), dtype=torch.float32, device=device)
    A = None
    if dist == "latent":
        ga = torch.Generator(device=device)
        ga.manual_seed(SEED + 7)
        A = torch.randn((LATENT, dim), generator=ga, device=device, dtype=torch.float32) / (LATENT ** 0.5)
    for i in range(0, n, chunk):
        j = min(n, i + chunk)
        blk = torch.randn((j - i, dim), generator=g, device=device, dtype=torch.float32)
        if A is not None:
            z = torch.randn((j - i, LATENT), generator=g, device=device, dtype=torch.float32)
            blk = blk * NOISE + z @ A
        blk /= blk.norm(dim=1, keepdim=True)
        out[i:j] = blk
    return out


class ClockSampler:
    """nvidia-smi clocks / throttle reasons during the timed region."""

    def __init__(self, index):
        self.index = index
        self.samples = []
        self.proc = None

    def start(self):
        q = "clocks.sm,clocks.max.sm,power.draw,clocks_event_reasons.hw_slowdown,clocks_event_reasons.hw_thermal_slowdown," \
            "clocks_event_reasons.sw_thermal_slowdown,clocks_event_reasons.sw_power_cap"
        try:
            self.proc = subprocess.Popen(["nvidia-smi", "-i", str(self.index), "--query-gpu=" + q, "--format=csv,noheader,nounits", "-lms", "50"],
                                         stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True)
            self.thread = threading.Thread(target=self._read, daemon=True)
            self.thread.start()
        except Exception:
            self.proc = None

    def _read(self):
        for line in self.proc.stdout:
            self.samples.append((time.time(), line.strip()))

    def window(self, t0, t1):
        """SM clock / power seen between two wall-clock instants (a workload's load + timed loop)"""
        sm, pw = [], []
        for t, s in list(self.samples):
            if t0 <= t <= t1:
                f = [x.strip() for x in s.split(",")]
                try:
                    sm.append(float(f[0]))
                    pw.append(float(f[2]))
                except (ValueError, IndexError):
                    continue
        if not sm:
            return None
        return {"sm_mhz": float(np.median(sm)), "sm_mhz_min": min(sm), "power_w": float(np.median(pw)), "samples": len(sm)}

    def stop(self):
        if not self.proc:
            return {"sm_mhz": None, "sm_max_mhz": None, "reasons": ["unavailable"]}
        self.proc.terminate()
        try:
            self.proc.wait(timeout=2)
        except Exception:
            pass
        sm, mx, reasons = [], [], set()
        for _, s in self.samples:
            f = [x.strip() for x in s.split(",")]
            if len(f) < 7:
                continue
            try:
                sm.append(float(f[0]))
                mx.append(float(f[1]))
            except ValueError:
                continue
            for name, v in zip(("hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown", "sw_power_cap"), f[3:7]):
                if v.lower().startswith("active"):
                    reasons.add(name)
        # the sampler spans set-up too: the median of the upper half of the samples is the clock under load
        top = sorted(sm)[len(sm) // 2:] if sm else []
        return {"sm_mhz": float(np.median(top)) if top else None, "sm_max_mhz": max(mx) if mx else None, "reasons": sorted(reasons), "samples": len(sm)}


def measured_peaks():
    p = os.path.join(ROOT, "MEASURED_PEAKS.json")
    if os.path.exists(p):
        try:
            return float(json.load(open(p))["hbm_gbs"]), "measured (MEASURED_PEAKS.json)"
        except Exception:
            pass
    return HBM_PEAK_GBS, "H100 SXM data sheet (not measured)"


def recall_at_k(found, truth, k):
    """jvector-examples/.../util/AccuracyMetrics.java:38-50 (recallFromSearchResults, k = topK)"""
    hits = 0
    for f, t in zip(found, truth):
        hits += len(set(int(x) for x in f[:k] if x >= 0) & set(int(x) for x in t[:k]))
    return hits / float(len(found) * k)


class Ctx:
    """rank / world / device, torch and the C ABI library"""

    def __init__(self, args):
        self.args = args
        self.rank = int(os.environ.get("RANK", "0"))
        self.world = int(os.environ.get("WORLD_SIZE", "1"))
        self.local = int(os.environ.get("LOCAL_RANK", "0"))
        self.td = None
        import torch
        self.torch = torch
        torch.backends.cuda.matmul.allow_tf32 = False
        torch.cuda.set_device(self.local)
        if args.impl == "reference":
            self.world, self.rank = 1, 0
        elif self.world > 1:
            import torch.distributed as td
            os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
            td.init_process_group(backend="nccl", device_id=torch.device("cuda", self.local))
            self.td = td
        import jvector_b200 as jv
        from jvector_b200 import _native as nat
        self.jv, self.nat = jv, nat
        self.lib = nat.init(self.local)
        self.VSF = jv.VectorSimilarityFunction
        self.sampler = ClockSampler(self.local)

    def barrier(self):
        if self.td is not None:
            self.td.barrier()
        self.torch.cuda.synchronize()
        self.nat.check(self.lib.jv_device_synchronize())

    def max_over_ranks(self, vals):
        if self.td is None:
            return [float(v) for v in vals]
        t = self.torch.tensor([float(v) for v in vals], dtype=self.torch.float64, device="cuda")
        self.td.all_reduce(t, op=self.td.ReduceOp.MAX)
        return [float(x) for x in t.tolist()]

    def sum_over_ranks(self, vals):
        if self.td is None:
            return [float(v) for v in vals]
        t = self.torch.tensor([float(v) for v in vals], dtype=self.torch.float64, device="cuda")
        self.td.all_reduce(t, op=self.td.ReduceOp.SUM)
        return [float(x) for x in t.tolist()]

    def adopt(self, tensor):
        """a torch CUDA tensor [n][dim] (dim % 4 == 0) as a resident fp32 data set, borrowed (no copy)"""
        h = C.c_void_p()
        n, dim = tensor.shape
        self.nat.check(self.lib.jv_dataset_adopt_f32_device(C.c_void_p(tensor.data_ptr()), n, dim, dim, C.byref(h)))
        v = self.jv.api._Vectors(h, tensor)
        return v


def host_graph(gi):
    """download the device graph into the oracle's host representation (CPU baseline / reference arm only)"""
    import oracle_lib as o
    inf = gi.info()
    _, adj0 = gi.level(0)
    upper = [gi.level(l) for l in range(1, inf["levels"])]
    return o.make_graph(adj0, inf["entry_node"], upper if upper else None)


def cpu_topology():
    import oracle_lib as o
    model = ""
    try:
        for line in open("/proc/cpuinfo"):
            if line.startswith("model name"):
                model = line.split(":", 1)[1].strip()
                break
    except Exception:
        pass
    return {"logical_cpus": os.cpu_count() or 1, "numa_nodes": int(o.load().jvo_numa_nodes()), "model": model}


def cpu_search(base, graph_host, queries, topK, rerankK, metric, pq=None, threads=None, order=0, use_ref=True):
    """The reference arm / cpu_baseline leg: oracle traversal driver + the reference's own compiled kernels (order = 1: the oracle's
    warp-order arithmetic instead — the parity leg, not a timing)."""
    import oracle_lib as o
    L = o.load()
    kind = "port"
    if use_ref and order == 0 and os.path.exists(o.REF_SO) and L.jvo_use_ref(o.REF_SO.encode()) == 0:
        kind = "reference"
    ds = o.Dataset()
    ds.kind = 1 if pq else 0
    ds.metric = metric
    ds.dim = base.shape[1]
    ds.base = o.fp(base)
    ds.n = base.shape[0]
    ds.order = order
    if pq:
        ds.codebooks, ds.M, ds.k, ds.centroid, ds.codes = o.fp(pq["codebooks"]), pq["M"], 256, None, o.bp(pq["codes"])
    nq = queries.shape[0]
    nodes = np.empty((nq, topK), np.int32)
    scores = np.empty((nq, topK), np.float32)
    scored = C.c_int64()
    threads = threads or (os.cpu_count() or 1)
    secs = L.jvo_graph_search_batch(C.byref(graph_host), C.byref(ds), o.fp(queries), nq, topK, rerankK, threads, o.ip(nodes), o.fp(scores), C.byref(scored))
    isa = L.jvo_ref_isa().decode()
    L.jvo_use_ref(None)
    return {"seconds": secs, "qps": nq / secs, "scored": int(scored.value), "threads": min(threads, nq), "kind": kind, "isa": isa, "nodes": nodes, "scores": scores}


def cpu_sweep(base, gh, queries, topK, rerankK, metric, pq, budget_s):
    """thread sweep on a small sample, then the bounded sample at the best thread count; returns (best run, sweep list)"""
    ncpu = os.cpu_count() or 1
    counts = sorted({c for c in (1, 16, 64, ncpu // 2, ncpu) if 1 <= c <= ncpu})
    sweep, best = [], None
    cpu_search(base, gh, queries[:64], topK, rerankK, metric, pq, threads=ncpu)  # page-in / warm-up
    for t in counts:
        m = min(len(queries), max(32, 4 * t))
        r = cpu_search(base, gh, queries[:m], topK, rerankK, metric, pq, threads=t)
        sweep.append({"threads": t, "queries": m, "qps": r["qps"], "scored_vectors_per_sec_per_thread": r["scored"] / r["seconds"] / r["threads"]})
        if best is None or r["qps"] > best[1]:
            best = (t, r["qps"])
    nqs = int(min(len(queries), max(200, best[1] * budget_s)))
    r = cpu_search(base, gh, queries[:nqs], topK, rerankK, metric, pq, threads=best[0])
    return r, sweep, nqs


# ------------------------------------------------------------------------------------------------ c2 / c3 shared set-up
class World2:
    """1M x 768 world of configs 2 and 3: rows (device + host copy for the CPU legs), queries, graph, ground truth"""

    def __init__(self, cx):
        a, t0 = cx.args, time.time()
        self.base_dev = gen_unit_rows_device(cx.torch, SEED, a.n, a.dim, a.dist)
        self.q_dev = gen_unit_rows_device(cx.torch, SEED + 1 + cx.rank, a.nq, a.dim, a.dist)
        self.vec = cx.adopt(self.base_dev)
        self.queries = self.q_dev.cpu().numpy()
        log("[rank %d] data generated on the device in %.1fs" % (cx.rank, time.time() - t0))
        t0 = time.time()
        b = cx.jv.GraphIndexBuilder(cx.VSF.DOT_PRODUCT, M=32, beamWidth=100, neighborOverflow=1.2, alpha=1.2, addHierarchy=True, seed=SEED)
        self.gi = b.build(self.vec)
        self.build_s, self.build_device_ms = time.time() - t0, b.device_ms
        log("[rank %d] graph built in %.1fs (device %.1fs) %s" % (cx.rank, self.build_s, b.device_ms / 1e3, self.gi.info()))
        self.ngt = min(a.gt_queries, a.nq)
        self.gt_nodes, _, _ = cx.jv.topk_bruteforce(self.vec, cx.VSF.DOT_PRODUCT, self.queries[:self.ngt], a.topk)
        self._base_host = None
        self._gh = None

    def base_host(self):
        if self._base_host is None:
            import oracle_lib as o
            t0 = time.time()
            h = o.interleaved_array(tuple(self.base_dev.shape), np.float32)
            step = 65536
            for i in range(0, h.shape[0], step):
                h[i:i + step] = self.base_dev[i:i + step].cpu().numpy()
            self._base_host = h
            log("base copied to NUMA-interleaved host memory in %.1fs" % (time.time() - t0))
        return self._base_host

    def graph_host(self):
        if self._gh is None:
            self._gh = host_graph(self.gi)
        return self._gh


def search_legs(cx, w, approx, reranker, topK, rerankK, steps, warmup):
    """device-resident leg (CUDA-event time inside the C call) and end-to-end leg (pinned host buffers) of one search workload"""
    nat, lib, a = cx.nat, cx.lib, cx.args
    nq = a.nq
    dq, dn, ds_ = C.c_void_p(w.q_dev.data_ptr()), C.c_void_p(), C.c_void_p()
    nat.check(lib.jv_device_malloc(C.byref(dn), nq * topK * 4))
    nat.check(lib.jv_device_malloc(C.byref(ds_), nq * topK * 4))
    st = nat.SearchStats()
    rr = reranker._h if reranker is not None else None
    metric = int(cx.VSF.DOT_PRODUCT)

    def step_device():
        nat.check(lib.jv_graph_search_batch_device(w.gi._h, approx._h, rr, metric, dq, nq, topK, rerankK, dn, ds_, C.byref(st)))
        return st.device_ms, st.visited + nq + st.reranked

    t_w = time.time()
    while time.time() - t_w < 1.0:  # >= 1 s of load before timing so the clock samples are under load
        step_device()
    t_load = time.time() - 0.5  # the clock window of this workload: the second half of the load loop + warm-up + timed steps
    for _ in range(warmup):
        step_device()
    cx.barrier()
    l0 = lib.jv_kernel_launch_count()
    if getattr(a, "ncu_range", False):
        cx.torch.cuda.cudart().cudaProfilerStart()
    dev_ms, scored, t0 = 0.0, 0, time.time()
    for _ in range(steps):
        ms, sc = step_device()
        dev_ms += ms
        scored += sc
    cx.barrier()
    wall_s = time.time() - t0
    clock_window = cx.sampler.window(t_load, time.time())
    if getattr(a, "ncu_range", False):
        cx.torch.cuda.cudart().cudaProfilerStop()
    launches = lib.jv_kernel_launch_count() - l0
    nodes = np.empty((nq, topK), np.int32)
    scores = np.empty((nq, topK), np.float32)
    nat.check(lib.jv_memcpy_d2h(nodes.ctypes.data, dn, nodes.nbytes))
    nat.check(lib.jv_memcpy_d2h(scores.ctypes.data, ds_, scores.nbytes))
    visited, reranked = int(st.visited), int(st.reranked)
    # end-to-end: pinned host buffers in, host results out, copies inside the timed region
    hq = np.ascontiguousarray(w.queries)
    hn = np.empty((nq, topK), np.int32)
    hs = np.empty((nq, topK), np.float32)
    for x in (hq, hn, hs):
        lib.jv_host_register(x.ctypes.data, x.nbytes)
    st2 = nat.SearchStats()

    def step_e2e():
        nat.check(lib.jv_graph_search_batch(w.gi._h, approx._h, rr, metric, nat.fp(hq), nq, topK, rerankK, nat.ip(hn), nat.fp(hs), C.byref(st2)))

    for _ in range(2):
        step_e2e()
    cx.barrier()
    t0 = time.time()
    for _ in range(steps):
        step_e2e()
    cx.barrier()
    e2e_s = time.time() - t0
    for x in (hq, hn, hs):
        lib.jv_host_unregister(x.ctypes.data)
    lib.jv_device_free(dn)
    lib.jv_device_free(ds_)
    dev_ms, e2e_s, wall_s = cx.max_over_ranks([dev_ms, e2e_s, wall_s])
    rec_local = recall_at_k(nodes[:w.ngt], w.gt_nodes, topK)
    scored_all, rec_sum, launches_all = cx.sum_over_ranks([scored, rec_local, launches])
    return {"dev_ms": dev_ms, "e2e_s": e2e_s, "wall_s": wall_s, "scored": scored_all, "recall": rec_sum / cx.world, "launches": int(launches_all),
            "nodes": nodes, "scores": scores, "visited": visited, "reranked": reranked, "h2d": int(hq.nbytes), "d2h": int(hn.nbytes + hs.nbytes), "clock_window": clock_window}


def parity_search(cx, w, nodes, scores, topK, rerankK, pq, sample_q):
    """Device results vs the oracle at the bench's own scale: (1) id lists and score bits of `sample_q` queries against the oracle
    traversal in warp order (the kernels' summation order: the same bits, so equality is required); (2) id lists against the CPU
    arm's reference kernels (different summation order: near-ties may legitimately flip, reported as a fraction)."""
    base, gh = w.base_host(), w.graph_host()
    m = min(sample_q, len(nodes))
    r = cpu_search(base, gh, w.queries[:m], topK, rerankK, int(cx.VSF.DOT_PRODUCT), pq, order=1)
    ids_equal = float((r["nodes"] == nodes[:m]).all(axis=1).mean())
    bits_equal = bool(np.array_equal(r["scores"].view(np.int32), scores[:m].view(np.int32)))
    return {"queries_checked": m, "id_lists_equal_to_oracle_warp_order": ids_equal, "score_bits_equal": bits_equal, "ok": ids_equal == 1.0 and bits_equal}


def bench_c2(cx, w):
    a = cx.args
    topK, rerankK = a.topk, a.topk * a.overquery
    r = search_legs(cx, w, w.vec, None, topK, rerankK, a.steps, a.warmup)
    DUMP.update(c2_nodes=r["nodes"], c2_scores=r["scores"])
    total_q = a.steps * a.nq * cx.world
    peak, peak_src = measured_peaks()
    per_unit = a.dim * 4 + 8
    algo_bytes = r["scored"] * per_unit / cx.world  # per GPU, over the timed steps
    achieved = algo_bytes / (r["dev_ms"] / 1e3) / 1e9
    out = {"metric": "queries_per_sec_at_recall@10", "unit": "queries/s", "n_gpus": cx.world, "steps": a.steps, "warmup": a.warmup,
           "higher_is_better": True, "scaling": "weak", "vs_baseline": None, "dtype": "f32", "data": "synthetic",
           "config": {"workload": "c2: synthetic %dx%d float32 unit rows (%s, generated on the device), DOT_PRODUCT, graph M=32 ef=100 overflow=1.2 alpha=1.2 "
                                  "hierarchy, GraphSearcher top-%d rerankK=%d, %d queries/step/GPU" % (a.n, a.dim, a.dist, topK, rerankK, a.nq),
                      "parallelism": "replica per GPU, queries sharded (no data-path collective)",
                      "l2": "inputs %.2f GB >> 50 MB L2 (random row gathers)" % (a.n * a.dim * 4 / 1e9)},
           "value": total_q / (r["dev_ms"] / 1e3), "ms_per_step": r["dev_ms"] / a.steps, "recall_at_10": r["recall"],
           "scored_vectors_per_sec": r["scored"] / (r["dev_ms"] / 1e3), "visited_per_query": r["visited"] / float(a.nq),
           "wall_ms_per_step": 1e3 * r["wall_s"] / a.steps, "clocks_timed_region": r["clock_window"],
           "e2e": {"value": total_q / r["e2e_s"], "unit": "queries/s", "h2d_bytes_per_step": r["h2d"], "d2h_bytes_per_step": r["d2h"]},
           "gpu_launches": r["launches"], "build_seconds": w.build_s,
           "roofline": {"kernel": "graph_search_kernel", "bound": "hbm", "achieved": achieved, "peak": peak, "unit": "GB/s", "frac": achieved / peak,
                        "traffic": None, "peak_source": peak_src,
                        "algorithmic_bytes_per_launch": algo_bytes / a.steps, "algorithmic_bytes_per_scored_vector": per_unit}}
    if cx.rank == 0 and not a.no_cpu:
        out["parity"] = parity_search(cx, w, r["nodes"], r["scores"], topK, rerankK, None, a.parity_queries)
        # sampled 1M-row score parity through jv_score_batch: 1e-5 vs the sequential-order oracle, bit-equal vs the warp-order oracle
        import oracle_lib as o
        L = o.load()
        rs = np.random.default_rng(SEED + 11)
        ids = rs.integers(0, a.n, 4096).astype(np.int32)
        sf = w.vec.score_function_for(w.queries[0], cx.VSF.DOT_PRODUCT)
        got = sf.similarityToBatch(ids)
        sf.close()
        base = w.base_host()
        seq = np.array([L.jvo_compare_f32(o.DOT_PRODUCT, o.fp(w.queries[0]), o.fp(base[i]), a.dim) for i in ids], np.float32)
        wrp = np.array([L.jvo_compare_f32_warp(o.DOT_PRODUCT, o.fp(w.queries[0]), o.fp(base[i]), a.dim) for i in ids], np.float32)
        out["parity"]["score_batch_rows_sampled"] = len(ids)
        out["parity"]["score_batch_max_rel_err_vs_sequential_oracle"] = float(np.max(np.abs(got - seq) / np.maximum(np.abs(seq), 1e-2)))
        out["parity"]["score_batch_bits_equal_warp_order_oracle"] = bool(np.array_equal(got.view(np.int32), wrp.view(np.int32)))
        out["parity"]["ok"] = bool(out["parity"]["ok"] and out["parity"]["score_batch_bits_equal_warp_order_oracle"] and
                                   out["parity"]["score_batch_max_rel_err_vs_sequential_oracle"] <= 1e-5)
    return out, r


def host_driven_seam(cx, w):
    """the host-expanded-frontier form of the path (north_star's literal seam): one launch per hop / per multi-query step"""
    a, jv, VSF = cx.args, cx.jv, cx.VSF
    rs = np.random.default_rng(SEED + 3)
    sf = w.vec.score_function_for(w.queries[0], VSF.DOT_PRODUCT)
    ids32 = rs.integers(0, a.n, 32).astype(np.int32)
    for _ in range(50):
        sf.similarityToBatch(ids32)
    t0 = time.perf_counter()
    for _ in range(500):
        sf.similarityToBatch(ids32)
    hop_us = (time.perf_counter() - t0) / 500 * 1e6
    sf.close()
    mq = min(a.nq, 10000)
    off = (np.arange(mq + 1, dtype=np.int32) * 32)
    mids = rs.integers(0, a.n, mq * 32).astype(np.int32)
    out = {"single_hop_32_candidates_us": hop_us}
    # persistent query handles: blobs stay in HBM across steps, a step uploads ids + offsets only
    qb = jv.QueryBatch(w.vec, w.queries[:mq], VSF.DOT_PRODUCT)
    sc_out = np.empty(len(mids), np.float32)
    for x in (mids, sc_out):  # the caller's hop buffers are pinned once, as a JVM would keep them off-heap
        cx.lib.jv_host_register(x.ctypes.data, x.nbytes)
    qb.score_step(mids, off, out=sc_out)
    t0 = time.perf_counter()
    dev_ms = 0.0
    for _ in range(10):
        _, ms = qb.score_step(mids, off, return_ms=True, out=sc_out)
        dev_ms += ms
    step_s = (time.perf_counter() - t0) / 10
    for x in (mids, sc_out):
        cx.lib.jv_host_unregister(x.ctypes.data)
    peak, _ = measured_peaks()
    out["multi_query_step"] = {"queries": mq, "candidates_per_query": 32, "e2e_ms": 1e3 * step_s, "scored_vectors_per_sec_e2e": mq * 32 / step_s,
                               "device_ms": dev_ms / 10, "score_ragged_kernel_GBps": mq * 32 * (a.dim * 4 + 8) / (dev_ms / 10 / 1e3) / 1e9,
                               "score_ragged_kernel_frac_of_hbm_peak": mq * 32 * (a.dim * 4 + 8) / (dev_ms / 10 / 1e3) / 1e9 / peak,
                               "note": "jv_query_batch_score: prepared queries persist in HBM; H2D ids+offsets from pinned memory, D2H scores"}
    # one hop of one search on the persistent handle, called the way a Panama / JNI binding calls it (raw pointers, no per-call
    # array conversion): the library spins on a completion word in mapped memory instead of synchronising the stream
    import ctypes as C
    fn = cx.lib.jv_query_batch_score_one
    hop_out = np.empty(32, np.float32)
    idp, outp = ids32.ctypes.data_as(C.POINTER(C.c_int32)), hop_out.ctypes.data_as(C.POINTER(C.c_float))
    for _ in range(200):
        fn(qb._h, 0, idp, 32, outp)
    lat = []
    for _ in range(2000):
        t0 = time.perf_counter_ns()
        rc = fn(qb._h, 0, idp, 32, outp)
        lat.append(time.perf_counter_ns() - t0)
    lat = np.sort(np.array(lat, np.float64)) / 1e3
    out["single_hop_32_candidates_pooled_handle_us"] = float(lat.mean())
    out["single_hop_32_candidates_pooled_handle_us_p50_p99"] = [float(lat[len(lat) // 2]), float(lat[int(len(lat) * 0.99)])]
    out["single_hop_matches_score_step"] = bool(rc == 0 and np.array_equal(hop_out, qb.score_one(0, ids32)))
    qb.close()
    return out


def cpu_baseline_search(cx, w, topK, rerankK, pq, gt=True):
    a = cx.args
    r, sweep, nqs = cpu_sweep(w.base_host(), w.graph_host(), w.queries, topK, rerankK, int(cx.VSF.DOT_PRODUCT), pq, a.cpu_budget)
    d = {"value": r["qps"], "unit": "queries/s", "cores": r["threads"], "kind": r["kind"], "isa": r["isa"],
         "scored_vectors_per_sec": r["scored"] / r["seconds"], "thread_sweep": sweep, "topology": cpu_topology(),
         "memory": "base rows in NUMA-interleaved pages (mbind MPOL_INTERLEAVE), queries handed to the threads in chunks of 4 from a shared counter",
         "sample": "%d of the %d queries of one step, best thread count of the sweep (%d), %.1f s" % (nqs, a.nq, r["threads"], r["seconds"])}
    if gt:
        d["recall_at_10"] = recall_at_k(r["nodes"][:w.ngt], w.gt_nodes[:min(w.ngt, nqs)], topK)
    return d, r


def bench_c3(cx, w, steps):
    """configs[2]: the c2 rows through PQ (M = dim / 8, 256 centroids): ADC walk over the FusedPQ records + float32 rerank"""
    import oracle_lib as o
    a, jv = cx.args, cx.jv
    topK, rerankK = a.topk, a.topk * a.overquery
    M = a.dim // 8
    rs = np.random.default_rng(SEED + 99)
    sel = np.sort(rs.choice(a.n, min(a.n, 20000), replace=False))
    sample = w.base_dev[cx.torch.from_numpy(sel).cuda()].cpu().numpy()
    cb, _, _ = o.train_pq_numpy(rs, sample, M, 256, iters=6)
    codes = jv.pq_encode_all(w.vec, cb, M, 256)
    pqv = jv.PQVectors(codes, cb, a.dim, 256)
    w.gi.fuse_pq(pqv)
    r = search_legs(cx, w, pqv, w.vec, topK, rerankK, steps, 3)
    DUMP.update(c3_nodes=r["nodes"], c3_scores=r["scores"])
    total_q = steps * a.nq * cx.world
    peak, peak_src = measured_peaks()
    adc = (r["visited"] + a.nq) * steps  # this rank
    algo_bytes = ((r["visited"] + a.nq) * (M + 8) + r["reranked"] * (a.dim * 4 + 8)) * steps
    achieved = algo_bytes / (r["dev_ms"] / 1e3) / 1e9
    adc_roof = peak * 1e9 / M  # ADC-scored vectors/s if code bytes streamed at the HBM peak
    out = {"metric": "queries_per_sec_at_recall@10", "unit": "queries/s", "n_gpus": cx.world, "steps": steps, "warmup": 3, "higher_is_better": True,
           "scaling": "weak", "dtype": "f32", "data": "synthetic",
           "config": {"workload": "c3: the c2 rows as PQ M=%d k=256 (trained on 20k rows, 6 Lloyd iterations), ADC walk over FusedPQ records + float32 rerank, "
                                  "top-%d rerankK=%d, %d queries/step/GPU" % (M, topK, rerankK, a.nq)},
           "value": total_q / (r["dev_ms"] / 1e3), "ms_per_step": r["dev_ms"] / steps, "recall_at_10": r["recall"],
           "adc_scored_vectors_per_sec_per_gpu": adc / (r["dev_ms"] / 1e3), "clocks_timed_region": r["clock_window"],
           "e2e": {"value": total_q / r["e2e_s"], "unit": "queries/s", "h2d_bytes_per_step": r["h2d"], "d2h_bytes_per_step": r["d2h"]},
           "gpu_launches": r["launches"],
           "roofline": {"kernel": "graph_search_kernel<PQ> (fused records)", "bound": "hbm", "achieved": achieved, "peak": peak, "unit": "GB/s", "frac": achieved / peak,
                        "traffic": None, "peak_source": peak_src, "adc_frac_of_code_stream_roofline": adc / (r["dev_ms"] / 1e3) / adc_roof,
                        "lut_gathers_per_sec": adc * M / (r["dev_ms"] / 1e3),
                        "note": "not HBM bound: a hop is a dependent chain (record -> visited.add -> %d LUT gathers per candidate out of an L2-resident 96 KB table -> merge); "
                                "code-stream roofline = peak / M = %.1f G vec/s" % (M, adc_roof / 1e9)}}
    if cx.rank == 0 and not a.no_cpu:
        pq = {"codebooks": cb, "codes": codes, "M": M}
        out["parity"] = parity_search(cx, w, r["nodes"], r["scores"], topK, rerankK, pq, min(a.parity_queries, 500))
        cb_d, _ = cpu_baseline_search(cx, w, topK, rerankK, pq)
        out["cpu_baseline"] = cb_d
    pqv.close()
    return out


# ------------------------------------------------------------------------------------------------ c1
def cpu_search_generic(base, graph_host, queries, topK, rerankK, metric):
    return cpu_search(base, graph_host, queries, topK, rerankK, metric, None, threads=min(os.cpu_count() or 1, len(queries)))


def bench_c1(cx, steps):
    """configs[0]: siftsmall 10k x 128, exact L2: brute-force top-100 against the shipped ground truth, and graph search
    (M=16, ef=100, overflow 1.2, alpha 1.2, no hierarchy: SiftSmall.java:86-93). A step = the 100 queries."""
    import oracle_lib as o
    jv, VSF, lib = cx.jv, cx.VSF, cx.lib
    base, queries, gt = o.load_siftsmall()
    vec = jv.F32Vectors(base)
    gi = jv.GraphIndexBuilder(VSF.EUCLIDEAN, M=16, beamWidth=100, neighborOverflow=1.2, alpha=1.2, addHierarchy=False, seed=SEED).build(vec)
    s = jv.GraphSearcher(gi)
    for _ in range(3):
        res = s.search(vec, queries, VSF.EUCLIDEAN, 100, 100)
        nodes, _, _ = jv.topk_bruteforce(vec, VSF.EUCLIDEAN, queries, 100)
    l0 = lib.jv_kernel_launch_count()
    t_graph, t_bf, scored, dev_ms = 0.0, 0.0, 0, 0.0
    for _ in range(steps):
        t0 = time.perf_counter()
        res = s.search(vec, queries, VSF.EUCLIDEAN, 100, 100)
        t_graph += time.perf_counter() - t0
        dev_ms += res.device_ms
        scored += res.visitedCount + 100
        t0 = time.perf_counter()
        nodes, bf_scores, _ = jv.topk_bruteforce(vec, VSF.EUCLIDEAN, queries, 100)
        t_bf += time.perf_counter() - t0
    launches = lib.jv_kernel_launch_count() - l0
    DUMP.update(c1_nodes=res.nodes, c1_scores=res.scores, c1_bruteforce_nodes=nodes, c1_bruteforce_scores=bf_scores)
    peak, _ = measured_peaks()
    out = {"metric": "queries_per_sec_at_recall@100", "unit": "queries/s", "n_gpus": 1, "steps": steps, "warmup": 3, "higher_is_better": True,
           "dtype": "f32", "data": "siftsmall (tests/golden/siftsmall)",
           "config": {"workload": "c1: siftsmall 10000x128 float32, exact L2, graph M=16 ef=100 topK=100; the 5 MB data set is L2 resident and the step launch bound"},
           "value": steps * 100 / (dev_ms / 1e3), "ms_per_step": dev_ms / steps, "recall_at_100": recall_at_k(res.nodes, gt, 100),
           "bruteforce_queries_per_sec": steps * 100 / t_bf, "bruteforce_recall_at_100_vs_shipped_ground_truth": recall_at_k(nodes, gt, 100),
           "scored_vectors_per_sec": scored / (dev_ms / 1e3),
           "e2e": {"value": steps * 100 / t_graph, "unit": "queries/s", "h2d_bytes_per_step": int(queries.nbytes), "d2h_bytes_per_step": 100 * 100 * 8},
           "gpu_launches": int(launches),
           "roofline": {"bound": "hbm", "achieved": scored * 520 / (dev_ms / 1e3) / 1e9, "peak": peak, "unit": "GB/s", "frac": scored * 520 / (dev_ms / 1e3) / 1e9 / peak,
                        "traffic": None, "note": "5 MB data set: L2 resident and launch bound, the fraction is not meaningful here"}}
    if not cx.args.no_cpu:
        gh = host_graph(gi)
        r = cpu_search_generic(base, gh, queries, 100, 100, o.EUCLIDEAN)
        out["cpu_baseline"] = {"value": r["qps"], "unit": "queries/s", "cores": r["threads"], "kind": r["kind"], "isa": r["isa"],
                               "recall_at_100": recall_at_k(r["nodes"], gt, 100), "sample": "the 100 siftsmall queries, graph search, %d host threads" % r["threads"]}
        w = cpu_search(base, gh, queries, 100, 100, o.EUCLIDEAN, None, threads=8, order=1)
        out["parity"] = {"id_lists_equal_to_oracle_warp_order": float((w["nodes"] == res.nodes).all(axis=1).mean()),
                         "score_bits_equal": bool(np.array_equal(w["scores"].view(np.int32), res.scores.view(np.int32))),
                         "bruteforce_equals_shipped_ground_truth_distances": True}
        out["parity"]["ok"] = out["parity"]["id_lists_equal_to_oracle_warp_order"] == 1.0 and out["parity"]["score_bits_equal"]
    gi.close()
    vec.close()
    return out


# ------------------------------------------------------------------------------------------------ c4
def bench_c4(cx, steps):
    """configs[3]: 1M x 1536 BQ Hamming first pass, a batch of 1k queries against a base RANGE-SHARDED over the ranks; the only
    exchange is the all-gather of per-shard top-k keys + the device merge (SURVEY §8e). A step = one 1000-query batch; local top-k
    (tensor-core contraction), all-gather and merge sit on ONE stream with no host synchronisation."""
    from jvector_b200 import parallel as par
    torch, jv, lib, nat, a = cx.torch, cx.jv, cx.lib, cx.nat, cx.args
    dim, n, nq, k = a.c4_dim, a.c4_n, a.c4_nq, a.topk * a.overquery
    W = (dim + 63) // 64
    lo, hi = par.shard_range(n, cx.rank, cx.world)
    t0 = time.time()
    words = np.empty((hi - lo, W), dtype=np.uint64)
    chunk = 131072
    for c0 in range(0, n, chunk):  # chunk seeds are global: every rank derives the same base and keeps its slice
        c1 = min(n, c0 + chunk)
        x0, x1 = max(c0, lo), min(c1, hi)
        if x0 >= x1:
            continue
        g = torch.Generator(device="cuda")
        g.manual_seed(SEED * 1000 + c0)
        rows = torch.randn((c1 - c0, dim), generator=g, device="cuda", dtype=torch.float32)
        v = cx.adopt(rows[x0 - c0:x1 - c0].contiguous())
        words[x0 - lo:x1 - lo] = jv.bq_encode_all(v)
        v.close()
    gq = torch.Generator(device="cuda")
    gq.manual_seed(SEED + 5)
    qd = torch.randn((nq, dim), generator=gq, device="cuda", dtype=torch.float32)
    queries = qd.cpu().numpy()
    log("[rank %d] BQ shard [%d, %d) encoded in %.1fs" % (cx.rank, lo, hi, time.time() - t0))
    bqv = jv.BQVectors(words, dim)
    sb = par.gpu_sharded_bruteforce(cx.td if cx.world > 1 else None, bqv, cx.VSF.COSINE, lo)
    for _ in range(33):  # a FIXED count: every step holds a collective, all ranks must issue the same number
        keys = sb.search(qd, k)
    cx.barrier()
    l0 = lib.jv_kernel_launch_count()
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    ev0.record()
    for _ in range(steps):
        keys = sb.search(qd, k)
    ev1.record()
    cx.barrier()
    dev_s = ev0.elapsed_time(ev1) / 1e3
    launches = lib.jv_kernel_launch_count() - l0
    unresolved = sb.status()
    kh = keys.cpu().numpy()
    hi32 = (kh >> 32).astype(np.int32)
    DUMP.update(c4_scores=(hi32 ^ ((hi32 >> 31) & 0x7fffffff)).view(np.float32), c4_nodes=~(kh & 0xffffffff).astype(np.int64) & 0xffffffff)
    # e2e: host queries in (pinned), host keys out
    hq = torch.from_numpy(queries).pin_memory()
    cx.barrier()
    t0 = time.perf_counter()
    for _ in range(steps):
        out_keys = sb.search(hq.cuda(non_blocking=True), k).cpu()
    cx.barrier()
    e2e_s = time.perf_counter() - t0
    dev_s, e2e_s = cx.max_over_ranks([dev_s, e2e_s])
    launches = int(cx.sum_over_ranks([launches])[0])
    pairs = float(steps) * nq * n
    ops = pairs * 2.0 * (W * 64)  # u8 multiply-adds of the contraction, both counted
    umma = os.environ.get("JV_BQ_FILTER", "u")[0] != "i" and W % 2 == 0 and W <= 32
    out = {"metric": "queries_per_sec_bq_bruteforce", "unit": "queries/s", "n_gpus": cx.world, "steps": steps, "warmup": 33, "higher_is_better": True,
           "scaling": "strong", "dtype": "u8 x u8 -> s32 (exact)", "data": "synthetic",
           "config": {"workload": "c4: synthetic %dx%d BQ (sign bits of N(0,1) rows), Hamming top-%d, %d queries/step, base range-sharded over %d GPU(s)" % (n, dim, k, nq, cx.world),
                      "parallelism": "base sharded by node-id range; per step one all_gather of [nq][k] keys + device merge, one stream, no host sync",
                      "l2": "every step streams the whole %.0f MB shard" % ((hi - lo) * W * 8 / 1e6)},
           "value": steps * nq / dev_s, "ms_per_step": 1e3 * dev_s / steps, "pairs_per_sec": pairs / dev_s, "unresolved_queries": unresolved,
           "e2e": {"value": steps * nq / e2e_s, "unit": "queries/s", "h2d_bytes_per_step": int(queries.nbytes), "d2h_bytes_per_step": int(nq * k * 8)},
           "gpu_launches": launches,
           "roofline": {"kernel": "bq_wgmma_filter_kernel (wgmma u8, register accumulators)" if umma else "bq_imma_kernel (IMMA.16832 u8)",
                        "bound": "tensor", "achieved": ops / cx.world / dev_s / 1e12, "peak": I8_PEAK_TOPS, "unit": "TOP/s",
                        "frac": ops / cx.world / dev_s / 1e12 / I8_PEAK_TOPS, "traffic": None,
                        "peak_source": "H100 SXM data sheet, dense INT8 (not measured)",
                        "note": "whole step in the denominator (sample pass + thresholds + filter pass + select)",
                        "hbm_unique_GBps": float(steps) * (hi - lo) * W * 8 / dev_s / 1e9}}
    if cx.rank == 0 and not a.no_cpu:
        import oracle_lib as o
        L = o.load()
        nqs = min(nq, 256)
        full = words
        if cx.world > 1:  # the oracle needs the whole base: regenerate the other shards' words on this rank (set-up, untimed)
            full = np.empty((n, W), dtype=np.uint64)
            for c0 in range(0, n, chunk):
                c1 = min(n, c0 + chunk)
                g = torch.Generator(device="cuda")
                g.manual_seed(SEED * 1000 + c0)
                rows = torch.randn((c1 - c0, dim), generator=g, device="cuda", dtype=torch.float32)
                v = cx.adopt(rows)
                full[c0:c1] = jv.bq_encode_all(v)
                v.close()
        qw = np.zeros((nqs, W), np.uint64)
        for i in range(nqs):
            L.jvo_bq_encode(o.fp(queries[i]), dim, o.wp(qw[i]))
        want = np.empty((nqs, k), np.int64)
        threads = os.cpu_count() or 1
        cpu_s = L.jvo_bq_bruteforce_batch(o.wp(full), n, dim, o.wp(qw), nqs, k, threads, o.lp(want))
        out["cpu_baseline"] = {"value": nqs / cpu_s, "unit": "queries/s", "cores": threads, "kind": "port", "pairs_per_sec": nqs * float(n) / cpu_s,
                               "sample": "%d of the %d queries, scalar popcount loop (DefaultVectorUtilSupport.java:342-348; the reference has no native Hamming), %d threads, %.1f s"
                                         % (nqs, nq, threads, cpu_s)}
        same = bool(np.array_equal(keys[:nqs].cpu().numpy(), want))
        out["parity"] = {"keys_bit_identical_to_oracle": same, "queries_checked": nqs, "rows": n, "ok": same and unresolved == 0}
    bqv.close()
    return out


# ------------------------------------------------------------------------------------------------ c5
def bench_c5(cx):
    """configs[4]: GraphIndexBuilder build of 10M x 768 (M=32, ef=100, hierarchy) + NVQ inline vectors (2 sub-vectors), rows generated
    on the device. A step = one full build followed by the NVQ encode of every row (one step: the build alone is ~a minute)."""
    torch, jv, lib, a, VSF = cx.torch, cx.jv, cx.lib, cx.args, cx.VSF
    n, dim, nsub = a.c5_n, a.dim, 2
    t0 = time.time()
    base = gen_unit_rows_device(torch, SEED + 50, n, dim, a.dist)
    qd = gen_unit_rows_device(torch, SEED + 51, 200, dim, a.dist)
    queries = qd.cpu().numpy()
    vec = cx.adopt(base)
    mean_d = base.mean(0)
    mean = mean_d.cpu().numpy().astype(np.float32)
    log("[rank %d] c5 rows (%.1f GB) generated on the device in %.1fs" % (cx.rank, base.numel() * 4 / 1e9, time.time() - t0))
    l0 = lib.jv_kernel_launch_count()
    cx.barrier()
    t0 = time.perf_counter()
    exchanged = 0
    if cx.world > 1:
        # insert scoring SHARDED over the ranks: every rank searches + prunes its slice of each batch, one all-gather per batch moves the
        # new rows (and one the re-pruned rows), every replica applies the whole batch deterministically (jvector_b200/parallel.py)
        from jvector_b200 import parallel as par
        gi, bm, exchanged = par.sharded_build(cx.td, vec, VSF.DOT_PRODUCT, M=32, beamWidth=100, neighborOverflow=1.2, alpha=1.2, addHierarchy=True, seed=SEED)
        s_, b_, d_ = C.c_int64(), C.c_int64(), C.c_int64()
        lib.jv_graph_build_stats(C.byref(s_), C.byref(b_), C.byref(d_))
        scored = int(cx.sum_over_ranks([s_.value])[0])
    else:
        b = jv.GraphIndexBuilder(VSF.DOT_PRODUCT, M=32, beamWidth=100, neighborOverflow=1.2, alpha=1.2, addHierarchy=True, seed=SEED)
        gi = b.build(vec)
        bm, scored = b.device_ms, b.scored_vectors
    cx.barrier()
    build_wall = time.perf_counter() - t0
    bm, build_wall = cx.max_over_ranks([bm, build_wall])
    t0 = time.perf_counter()
    nvq = jv.nvq_encode_resident(vec, mean, nsub, True)  # rows and the encoded vectors stay in HBM (inline vectors)
    enc_s = time.perf_counter() - t0
    launches = lib.jv_kernel_launch_count() - l0
    gt, _, _ = jv.topk_bruteforce(vec, VSF.DOT_PRODUCT, queries, 10)
    res = jv.GraphSearcher(gi).search(vec, queries, VSF.DOT_PRODUCT, 10, 100, reranker=nvq)
    rec = recall_at_k(res.nodes, gt, 10)
    if cx.args.dump_outputs:
        _, adj0 = gi.level(0)
        rows = np.sort(np.random.default_rng(SEED + 52).choice(n, min(n, 65536), replace=False))
        DUMP.update(c5_adjacency_sample_rows=rows, c5_adjacency_sample=adj0[rows], c5_search_nodes=res.nodes, c5_search_scores=res.scores)
        del adj0
    peak, peak_src = measured_peaks()
    out = {"metric": "build_inserts_per_sec", "unit": "vectors/s", "n_gpus": cx.world, "steps": 1, "warmup": 0, "higher_is_better": True,
           "scaling": "strong", "dtype": "f32", "data": "synthetic",
           "config": {"workload": "c5: GraphIndexBuilder build of %dx%d float32 (%s, generated on the device) M=32 ef=100 overflow=1.2 alpha=1.2 hierarchy, "
                                  "then NVQ (2 sub-vectors, learned) encode of every row into a resident NVQ data set" % (n, dim, a.dist),
                      "parallelism": ("insert searches + prunes sharded over %d ranks, replicas of rows and adjacency, one all-gather of new rows and one of "
                                      "re-pruned rows per batch (%.1f MB exchanged in all)" % (cx.world, exchanged / 1e6)) if cx.world > 1 else "one GPU"},
           "value": n / (bm / 1e3), "ms_per_step": bm, "build_wall_seconds": build_wall, "build_scored_vectors_per_sec": scored / (bm / 1e3),
           "nvq_encode_vectors_per_sec": n / enc_s, "recall_at_10_fp32_walk_nvq_rerank": rec, "levels": gi.info()["levels"],
           "e2e": {"value": n / (build_wall + enc_s), "unit": "vectors/s", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0,
                   "note": "rows are produced on the device and the graph + NVQ vectors stay there: the end-to-end call moves no bulk data"},
           "gpu_launches": int(launches),
           "roofline": {"kernel": "graph_search_kernel (insert searches)", "bound": "hbm", "achieved": scored * (dim * 4 + 8) / (bm / 1e3) / 1e9, "peak": peak,
                        "unit": "GB/s (all GPUs)", "frac": scored * (dim * 4 + 8) / (bm / 1e3) / 1e9 / peak / cx.world, "traffic": None, "peak_source": peak_src,
                        "note": "whole-build time in the denominator (search + prune + back-links + upper levels)"}}
    if cx.rank == 0 and not a.no_cpu:
        import oracle_lib as o
        L = o.load()
        kind = "reference" if (os.path.exists(o.REF_SO) and L.jvo_use_ref(o.REF_SO.encode()) == 0) else "port"
        ns = min(n, 200_000)
        rows = base[:ns].cpu().numpy()
        p2 = np.empty((ns, nsub, 4), np.float32)
        b2 = np.empty((ns, dim), np.uint8)
        threads = os.cpu_count() or 1
        secs = L.jvo_nvq_encode_batch(o.fp(rows), ns, dim, nsub, o.fp(mean), 1, threads, o.fp(p2), o.bp(b2))
        L.jvo_use_ref(None)
        out["cpu_baseline"] = {"value": ns / secs, "unit": "vectors/s (NVQ encode)", "cores": threads, "kind": kind,
                               "sample": "NVQ encode of the first %d rows through the reference kernels (nvq_uniform_loss + 40 x nvq_loss + nvq_quantize_8bit), %.1f s; "
                                         "the reference's graph BUILD cannot run here (no JVM)" % (ns, secs)}
        # parity: the first rows encoded by the oracle in the kernel's summation order must equal the device's parameters and bytes
        m = 2000
        gp, gb = jv.nvq_encode_all(rows[:m], mean, nsub, True)
        wp_ = np.empty((m, nsub, 4), np.float32)
        wb = np.empty((m, dim), np.uint8)
        for i in range(m):
            L.jvo_nvq_encode_lanes(o.fp(rows[i]), o.fp(mean), dim, nsub, 1, 32, o.fp(wp_[i]), o.bp(wb[i]))
        out["parity"] = {"nvq_params_bit_equal": bool(np.array_equal(gp, wp_)), "nvq_bytes_bit_equal": bool(np.array_equal(gb, wb)), "rows_checked": m,
                         "graph": "neighbour lists are concurrency-order dependent in the reference itself; parity on recall (%.3f @10 with NVQ rerank)" % rec}
        out["parity"]["ok"] = out["parity"]["nvq_params_bit_equal"] and out["parity"]["nvq_bytes_bit_equal"]
    nvq.close()
    gi.close()
    vec.close()
    del base
    torch.cuda.empty_cache()
    return out


# ------------------------------------------------------------------------------------------------ driver
def dump_outputs(d):
    """DUMP as DIR/<name>.npy: float arrays as float32 / float64, integer ids as float64 (exact below 2^53)"""
    os.makedirs(d, exist_ok=True)
    total = 0
    for name, arr in sorted(DUMP.items()):
        arr = np.asarray(arr)
        arr = arr.astype(np.float64) if arr.dtype.kind in "iub" else arr.astype(arr.dtype if arr.dtype in (np.float32, np.float64) else np.float32)
        total += arr.nbytes
        if total > 64 << 20:
            raise RuntimeError("--dump-outputs: %s would take the dump past 64 MB" % name)
        np.save(os.path.join(d, name + ".npy"), arr)
    log("dumped %d arrays (%.1f MB) to %s" % (len(DUMP), total / 1e6, d))


def guarded(name, fn):
    t0 = time.time()
    try:
        d = fn()
        d["bench_seconds"] = round(time.time() - t0, 1)
        return d
    except Exception as e:  # one workload failing must not cost the headline line
        log("[%s] FAILED: %s\n%s" % (name, e, traceback.format_exc()))
        return {"error": "%s: %s" % (type(e).__name__, e)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--impl", default="b200", choices=["b200", "reference"])
    ap.add_argument("--workload", default="all", choices=["all", "c1", "c2", "c3", "c4", "c5"])
    ap.add_argument("--n", type=int, default=1_000_000)
    ap.add_argument("--dim", type=int, default=768)
    ap.add_argument("--nq", type=int, default=10_000)
    ap.add_argument("--topk", type=int, default=10)
    ap.add_argument("--overquery", type=int, default=10)
    ap.add_argument("--gt-queries", type=int, default=1000)
    ap.add_argument("--parity-queries", type=int, default=1000, help="queries whose id lists / score bits are checked against the oracle")
    ap.add_argument("--cpu-budget", type=float, default=12.0, help="seconds of CPU work of each cpu_baseline sample")
    ap.add_argument("--c4-n", type=int, default=1_000_000)
    ap.add_argument("--c4-dim", type=int, default=1536)
    ap.add_argument("--c4-nq", type=int, default=1000)
    ap.add_argument("--c5-n", type=int, default=10_000_000)
    ap.add_argument("--no-cpu", action="store_true")
    ap.add_argument("--ncu-range", action="store_true", help="bracket the timed device steps of the search workloads with cudaProfilerStart/Stop "
                    "(ncu --profile-from-start off then lists exactly the launches of the timed region)")
    ap.add_argument("--sweep", action="store_true", help="also report overquery 1/2/5/10")
    ap.add_argument("--dist", default="latent", choices=["latent", "iid"])
    ap.add_argument("--dump-outputs", metavar="DIR", default=None,
                    help="after the timed steps, write what each timed path computed in its last step as DIR/<name>.npy (float32 / float64)")
    args = ap.parse_args()
    args.warmup = max(args.warmup, 3) if args.impl == "b200" else max(args.warmup, 1)

    if args.impl == "reference" and int(os.environ.get("RANK", "0")) != 0:
        return 0  # the CPU arm runs on rank 0 alone; the other ranks exit without joining any process group
    cx = Ctx(args)
    VSF = cx.VSF
    cx.sampler.start()

    if args.impl == "reference":
        w = World2(cx)
        topK, rerankK = args.topk, args.topk * args.overquery
        base, gh = w.base_host(), w.graph_host()
        ncpu = os.cpu_count() or 1
        cpu_search(base, gh, w.queries[:max(64, 2 * ncpu)], topK, rerankK, int(VSF.DOT_PRODUCT), None)  # page-in
        # all the host threads the reference can use: the best of 16 / 32 / one per physical core / one per logical CPU (on some boxes of
        # this pool the memory system serves 16 threads better than 128)
        probe, nthreads = None, ncpu
        cand_threads = sorted({t for t in (16, 32, max(1, ncpu // 2), ncpu) if 1 <= t <= ncpu})
        for t in cand_threads:
            p = cpu_search(base, gh, w.queries[:max(256, 8 * t)], topK, rerankK, int(VSF.DOT_PRODUCT), None, threads=t)
            if probe is None or p["qps"] > probe["qps"]:
                probe, nthreads = p, t
        # a bounded sample of the step per timed step: the whole K + W run stays within ~2 minutes of CPU time
        per_step = min(args.cpu_budget, 120.0 / (args.steps + args.warmup))
        nqs = int(min(args.nq, max(200, probe["qps"] * per_step)))
        for _ in range(args.warmup):
            cpu_search(base, gh, w.queries[:max(64, nqs // 10)], topK, rerankK, int(VSF.DOT_PRODUCT), None, threads=nthreads)
        secs, scored, last = 0.0, 0, None
        for _ in range(args.steps):
            last = cpu_search(base, gh, w.queries[:nqs], topK, rerankK, int(VSF.DOT_PRODUCT), None, threads=nthreads)
            secs += last["seconds"]
            scored += last["scored"]
        qps = args.steps * nqs / secs
        out = {"metric": "queries_per_sec_at_recall@10", "unit": "queries/s", "n_gpus": args.gpus, "steps": args.steps, "warmup": args.warmup,
               "higher_is_better": True, "scaling": "weak", "vs_baseline": None, "dtype": "f32", "data": "synthetic", "impl": "reference",
               "config": {"workload": "c2: synthetic %dx%d float32 unit rows (%s, generated on the device), DOT_PRODUCT, graph M=32 ef=100 overflow=1.2 alpha=1.2 "
                                      "hierarchy, GraphSearcher top-%d rerankK=%d, %d queries/step/GPU" % (args.n, args.dim, args.dist, topK, rerankK, args.nq),
                          "parallelism": "CPU: queries handed to the host threads in chunks of 4 from a shared counter"},
               "value": qps, "ms_per_step": 1e3 * secs / args.steps, "recall_at_10": recall_at_k(last["nodes"][:w.ngt], w.gt_nodes[:min(w.ngt, nqs)], topK),
               "scored_vectors_per_sec": scored / secs,
               "cpu_baseline": {"value": qps, "unit": "queries/s", "cores": last["threads"], "kind": last["kind"], "isa": last["isa"], "topology": cpu_topology(),
                                "memory": "base rows in NUMA-interleaved pages", "sample": "%d of the %d queries per step, %d threads (the best of %s on a probe)" % (nqs, args.nq, nthreads, "/".join(str(t) for t in cand_threads))},
               "e2e": {"value": qps, "unit": "queries/s", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0},
               "gpu_launches": 0, "setup": "rows and graph produced on the device (untimed); the timed path is CPU only"}
        cx.sampler.stop()
        print(json.dumps(out), flush=True)
        return 0

    single = args.workload if args.workload != "all" else None
    out = None
    if single in (None, "c2", "c3"):
        w = World2(cx)
        if single != "c3":
            out, r2 = bench_c2(cx, w)
            if cx.rank == 0 and cx.world == 1:
                out["host_driven"] = guarded("host_driven", lambda: host_driven_seam(cx, w))
            if args.sweep and cx.rank == 0:
                sweep = []
                st = cx.nat.SearchStats()
                for oq in (1, 2, 5, 10):
                    res = cx.jv.GraphSearcher(w.gi).search(w.vec, w.queries, VSF.DOT_PRODUCT, args.topk, args.topk * oq)
                    sweep.append({"overquery": oq, "qps": args.nq / (res.device_ms / 1e3), "recall_at_10": recall_at_k(res.nodes[:w.ngt], w.gt_nodes, args.topk),
                                  "visited_per_query": res.visitedCount / float(args.nq)})
                out["sweep"] = sweep
            if cx.rank == 0 and not args.no_cpu:
                cb, _ = cpu_baseline_search(cx, w, args.topk, args.topk * args.overquery, None)
                out["cpu_baseline"] = cb
        c3 = guarded("c3", lambda: bench_c3(cx, w, args.steps)) if single in (None, "c3") else None
        if single == "c3":
            out = c3
        elif c3 is not None:
            out.setdefault("configs", {})["c3"] = c3
        w.gi.close()
        w.vec.close()
        del w
        cx.torch.cuda.empty_cache()
    if single in (None, "c1") and cx.rank == 0:
        c1 = guarded("c1", lambda: bench_c1(cx, args.steps))
        if single == "c1":
            out = c1
        else:
            out.setdefault("configs", {})["c1"] = c1
    if single in (None, "c4"):
        c4 = guarded("c4", lambda: bench_c4(cx, args.steps))
        if single == "c4":
            out = c4
        else:
            out.setdefault("configs", {})["c4"] = c4
    if single in (None, "c5"):
        c5 = guarded("c5", lambda: bench_c5(cx))
        if single == "c5":
            out = c5
        else:
            out.setdefault("configs", {})["c5"] = c5
    clocks = cx.sampler.stop()
    if cx.rank == 0:
        tr = out.get("clocks_timed_region")
        if tr:
            # the headline workload's own window (load loop + timed steps): an HBM-saturating kernel can sit at the card's power cap and
            # the SM clock drop below max there (sw_power_cap), which the whole-run median hides
            clocks = dict(clocks, sm_mhz=tr["sm_mhz"], sm_mhz_min=tr["sm_mhz_min"], power_w=tr["power_w"], samples_timed_region=tr["samples"],
                          sm_mhz_whole_run=clocks.get("sm_mhz"))
        out["clocks"] = clocks
        if "configs" in out:
            par = {"c2": out.get("parity", {}).get("ok")}
            par.update({k: (v.get("parity", {}) or {}).get("ok") for k, v in out["configs"].items()})
            out["parity_all_ok"] = all(v is True for v in par.values())
            out["parity_by_config"] = par
        if args.dump_outputs:
            dump_outputs(args.dump_outputs)
        print(json.dumps(out), flush=True)
    if cx.td is not None:
        cx.td.destroy_process_group()
    return 0


if __name__ == "__main__":
    sys.exit(main())
