"""jv_graph_compact_pq restated on the host, on top of compact_model's fp32 merge: OnDiskGraphIndexCompactor with FusedPQ or sidecar
sources, and PQRetrainer's sample.

A source is compact_model's dict plus pq: a dict of codes [n][M] uint8, codebooks [k * dim], M, k and centroid (or None).

The fused form searches another source t as OnDiskGraphIndexCompactor.buildCrossSourceScoreProvider does, with t's own PQ: at level 0
a walk of t's FusedPQ records (the oracle's PQ scorer over the packed neighbour codes, jvo_fused_pq_pack of t's adjacency), above it
a walk of the members' plain code rows; each reranks its K survivors exactly over t's rows, both scorers in warp order. Everything
else (candidates, prune, levels, entry) is compact_model.compact, which runs here with this search in place of its exact one. The
sidecar form is compact_model.compact itself.

retrain_sample is PQRetrainer.sampleBalanced (PQRetrainer.java:127-212) with counter_random(seed, TAG_COMPACT_SAMPLE, source, i) in
place of ThreadLocalRandom."""
import contextlib
import ctypes as C

import numpy as np

import compact_model as cm
import oracle_lib as o
import pq_train_model as ptm
from oracle_lib import bp, fp, ip

MAX_PQ_TRAINING_SET_SIZE, MIN_SAMPLES_PER_SOURCE, SAMPLE_CHUNK_SIZE = 128000, 1000, 32
TAG_COMPACT_SAMPLE = 0x7ffffffe  # common.cuh


def chunk_order(seed, s, chunks):
    """source s's chunk order: Fisher-Yates over counter_random(seed, TAG_COMPACT_SAMPLE, s, i) % (i + 1), i = chunks - 1 .. 1"""
    order = list(range(chunks))
    for i in range(chunks - 1, 0, -1):
        j = int(ptm.counter_random(seed, TAG_COMPACT_SAMPLE, s, i)[0] % np.uint64(i + 1))
        order[i], order[j] = order[j], order[i]
    return order


def sample_quotas(live_counts, cap=MAX_PQ_TRAINING_SET_SIZE):
    """sampleBalanced's quotas for sources of these live counts (None: every live node is taken)"""
    S, total = len(live_counts), sum(live_counts)
    if total <= cap:
        return None
    lo = min(MIN_SAMPLES_PER_SOURCE, cap // S)
    quota = [max(lo, cap * int(c) // total) for c in live_counts]
    assigned = sum(quota)
    while assigned > cap:
        for s in range(S):
            if assigned <= cap:
                break
            if quota[s] > lo:
                quota[s] -= 1
                assigned -= 1
    while assigned < cap:
        for s in range(S):
            if assigned >= cap:
                break
            quota[s] += 1
            assigned += 1
    return quota


def retrain_sample(sources, seed, cap=MAX_PQ_TRAINING_SET_SIZE):
    """PQRetrainer.sampleBalanced: per source its sampled node ids, ascending"""
    live = [np.asarray(s["live"], bool) for s in sources]
    quota = sample_quotas([int(m.sum()) for m in live], cap)
    if quota is None:
        return [np.flatnonzero(m).astype(np.int32) for m in live]
    out = []
    for s, m in enumerate(live):
        n = len(m)
        taken = []
        for c in chunk_order(seed, s, -(-n // SAMPLE_CHUNK_SIZE)):
            if len(taken) >= quota[s]:
                break
            nodes = np.flatnonzero(m[c * SAMPLE_CHUNK_SIZE:(c + 1) * SAMPLE_CHUNK_SIZE]) + c * SAMPLE_CHUNK_SIZE
            taken.extend(nodes[:quota[s] - len(taken)].tolist())
        out.append(np.array(sorted(taken), np.int32))
    return out


def pq_sub_search(oracle, metric, src, level, queries, K):
    """compact_model.sub_search's K best live members of src's level `level`, walked over src's PQ codes (its FusedPQ records at level
    0) and reranked exactly over its rows"""
    ids, adj = cm.members(src, level)
    pos = np.full(src["adj0"].shape[0], -1, np.int64)
    pos[ids] = np.arange(len(ids))

    def remap(a):
        a = np.asarray(a, np.int64)
        return np.ascontiguousarray(np.where(a >= 0, pos[np.clip(a, 0, None)], -1), np.int32)

    upper = [(remap(i), remap(a)) for i, a in src["upper"][level:]]
    g = o.make_graph(remap(adj), int(pos[src["entry"]]), upper or None)
    rows = np.ascontiguousarray(src["data"][ids], np.float32)
    accept = cm._bits(src["live"][ids])
    n, dim = rows.shape
    pq = src["pq"]
    codes = np.ascontiguousarray(pq["codes"][ids], np.uint8)
    cb, cen, M = np.ascontiguousarray(pq["codebooks"], np.float32), pq["centroid"], pq["M"]
    degree = adj.shape[1]
    if level == 0:
        packed = np.empty((n, degree, M), np.uint8)
        oracle.jvo_fused_pq_pack(ip(np.ascontiguousarray(adj, np.int32)), n, degree, bp(codes), M, bp(packed))
    out = np.full((len(queries), K), -1, np.int32)
    for i, q in enumerate(queries):
        q = np.ascontiguousarray(q, np.float32)
        sf = oracle.jvo_scorer_pq(metric, fp(cb), M, pq["k"], dim, fp(cen) if cen is not None else None, bp(codes), n, fp(q))
        if level == 0:
            oracle.jvo_scorer_set_packed_neighbors(sf, bp(packed), degree)
        oracle.jvo_scorer_set_order(sf, 1)
        rr = oracle.jvo_scorer_f32(metric, fp(rows), n, dim, fp(q))
        oracle.jvo_scorer_set_order(rr, 1)
        nodes = np.full(K, -1, np.int32)
        scores = np.zeros(K, np.float32)
        oracle.jvo_graph_search_ex(C.byref(g), sf, rr, K, K, 0.0, 0.0, accept.ctypes.data_as(C.POINTER(C.c_uint32)), ip(nodes), fp(scores), None)
        oracle.jvo_scorer_free(sf)
        oracle.jvo_scorer_free(rr)
        out[i] = np.where(nodes >= 0, ids[np.clip(nodes, 0, None)], -1)
    return out


@contextlib.contextmanager
def _searching_pq():
    """compact_model.compact with pq_sub_search as its search of the other sources (its only change in the fused form)"""
    exact = cm.sub_search
    cm.sub_search = pq_sub_search
    try:
        yield
    finally:
        cm.sub_search = exact


def compact(oracle, metric, sources, alpha=1.2, fused=True):
    """compact_model.compact's result, with the other sources searched over their PQ when fused"""
    if not fused:
        return cm.compact(oracle, metric, sources, alpha)
    with _searching_pq():
        return cm.compact(oracle, metric, sources, alpha)


def compact_pq(oracle, metric, sources, seed, alpha=1.2, fused=True):
    """jv_graph_compact_pq: the merge (fused or sidecar) plus "sample" (per source its sampled nodes) and "train_rows" (the sampled
    rows in (source, node) order), on which source 0's codebooks are refined"""
    res = compact(oracle, metric, sources, alpha, fused)
    res["sample"] = retrain_sample(sources, seed)
    res["train_rows"] = np.concatenate([s["data"][x] for s, x in zip(sources, res["sample"])]).astype(np.float32)
    return res
