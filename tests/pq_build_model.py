"""The device graph build over PQ codes (jv_graph_build_pq, build.cu prune_kernel<.., KIND_PQ>) restated on the host, as the checker
of jv_builder_create_pq + jv_builder_*.

It is build_model.BuildModel with the scores of BuildScoreProvider.pqBuildScoreProvider:
  query   : decode(c_v) — per sub-space the codebook row plus the global centroid, one fp32 add per element
  search  : the oracle's warp-order traversal (jvo_graph_search) with jvo_scorer_pq over decode(c_v) in the kernels' order
            (jvo_scorer_set_order 1): the walk's own bits, no rerank, topK = rerankK = beam
  keys    : the same scorer's score of every candidate
  pairs   : pair_pq_table (scorers.cuh) restated in float32 over a given centroid-pair table: lane l sums the entries of sub-spaces
            m = l, l + 32, ... in increasing m, then the xor butterfly 16, 8, 4, 2, 1; cosine sum / sqrt(n1 n2); the score map last
  prune   : prune_kernel's selection restated literally (running maxima, alpha passes, the early drop at alpha_max)
Every score is the device's own bits, so nothing is flagged: any difference from the device is a bug."""
import ctypes as C

import numpy as np

import build_model as bm
import oracle_lib as o
from oracle_lib import bp, fp, ip

F32 = np.float32


def decode(codes, codebooks, sizes, offsets, k, centroid):
    """ProductQuantization.decode for every row of codes [n][M]: float32 [n][dim], the centroid added in one fp32 add"""
    n, M = codes.shape
    dim = int(sizes.sum())
    out = np.empty((n, dim), F32)
    for m in range(M):
        sz, off = int(sizes[m]), int(offsets[m])
        cb = codebooks[k * off:k * (off + sz)].reshape(k, sz)
        out[:, off:off + sz] = cb[codes[:, m]]
    if centroid is not None:
        out = (out + centroid[None, :]).astype(F32)
    return out


def tri_index(a, b, k):
    r, c = np.minimum(a, b).astype(np.int64), np.maximum(a, b).astype(np.int64)
    return r * k - (r * (r - 1) // 2) + (c - r)


def _warp_sum(terms):
    """terms [M][...] float32 -> pair_pq_table's order: lane partial sums over m = lane mod 32 in increasing m, xor butterfly"""
    M = terms.shape[0]
    lanes = np.zeros((32,) + terms.shape[1:], F32)
    for m in range(M):
        lanes[m % 32] = (lanes[m % 32] + terms[m]).astype(F32)
    for sh in (16, 8, 4, 2, 1):
        lanes = (lanes + lanes[np.arange(32) ^ sh]).astype(F32)
    return lanes[0]


def pair_scores(metric, table, k, ca, cb):
    """pair_pq_table for code rows ca [na][M] against cb [nb][M]: float32 [na][nb]. table: [M * k (k + 1) / 2], the squared-L2 table
    for EUCLIDEAN, the dot-product table otherwise (jv_dataset_pq_pair_table)"""
    M = ca.shape[1]
    block = k * (k + 1) // 2
    T = np.asarray(table, F32).reshape(M, block)

    def gather(x, y):
        return np.stack([T[m][tri_index(x[:, m][:, None], y[:, m][None, :], k)] for m in range(M)])

    s = _warp_sum(gather(ca, cb))
    if metric == o.COSINE:
        n1 = _warp_sum(np.stack([T[m][tri_index(ca[:, m], ca[:, m], k)] for m in range(M)]))
        n2 = _warp_sum(np.stack([T[m][tri_index(cb[:, m], cb[:, m], k)] for m in range(M)]))
        s = (s / np.sqrt((n1[:, None] * n2[None, :]).astype(F32))).astype(F32)
    if metric == o.EUCLIDEAN:
        return (F32(1) / (F32(1) + s)).astype(F32)
    return ((F32(1) + s) / F32(2)).astype(F32)


def prune_select(keys_scores, cands, P, degree, alpha):
    """prune_kernel's selection over candidates already in key order (score descending, lower id first): selected positions"""
    nc = len(cands)
    maxsim = np.full(nc, F32(-3.0e38), F32)
    state = np.zeros(nc, np.int8)  # 0 eligible, 1 selected, 2 dropped
    lim = F32(F32(alpha) + F32(1e-6))
    amax, a = F32(1.0), F32(1.0)
    while a <= lim:
        amax = a
        a = F32(a + F32(0.2))
    nsel = 0
    a = F32(1.0)
    while a <= lim and nsel < degree:
        cursor = 0
        while nsel < degree:
            pick = -1
            for i in range(cursor, nc):
                if state[i] == 0 and not maxsim[i] > F32(keys_scores[i] * a):
                    pick = i
                    break
            if pick < 0:
                break
            state[pick] = 1
            nsel += 1
            cursor = pick + 1
            if nsel >= degree:
                break
            live = state == 0
            maxsim[live] = np.maximum(maxsim[live], P[live, pick])
            drop = live & (maxsim > (keys_scores * amax).astype(F32))
            state[drop] = 2
        a = F32(a + F32(0.2))
    return [int(cands[i]) for i in range(nc) if state[i] == 1]


class PQBuildModel(bm.BuildModel):
    def __init__(self, oracle, codes, codebooks, k, dim, centroid, table, metric, M, beam, **kw):
        self.codes = np.ascontiguousarray(codes, np.uint8)
        self.codebooks = np.ascontiguousarray(codebooks, F32).reshape(-1)
        self.k, self.pq_m = k, self.codes.shape[1]
        self.centroid = None if centroid is None else np.ascontiguousarray(centroid, F32)
        self.table = np.ascontiguousarray(table, F32)
        self.sizes, self.offsets = o.pq_layout(dim, self.pq_m)
        self.queries = decode(self.codes, self.codebooks, self.sizes, self.offsets, k, self.centroid)
        super().__init__(oracle, self.queries, metric, M, beam, **kw)

    def scorer(self, v):
        """the warp-order PQ scorer of decode(c_v) (the caller frees it)"""
        sf = self.L.jvo_scorer_pq(self.metric, fp(self.codebooks), self.pq_m, self.k, self.dim, fp(self.centroid), bp(self.codes), self.n,
                                  fp(self.queries[v]))
        self.L.jvo_scorer_set_order(sf, 1)
        return sf

    def search(self, u):
        g = o.make_graph(self.adj, 0)
        sf = self.scorer(u)
        nodes = np.full(self.beam, -1, np.int32)
        scores = np.zeros(self.beam, F32)
        cnt = self.L.jvo_graph_search(C.byref(g), sf, None, self.beam, self.beam, ip(nodes), fp(scores), None)
        self.L.jvo_scorer_free(sf)
        return [int(x) for x in nodes[:cnt] if x >= 0]

    def key_scores(self, v, ids):
        sf = self.scorer(v)
        out = np.array([self.L.jvo_scorer_score(sf, int(i)) for i in ids], F32)
        self.L.jvo_scorer_free(sf)
        return out

    def prune(self, v, cands):
        c = np.array(sorted(set(int(x) for x in cands) - {int(v)}), dtype=np.int64)
        self.prunes += 1
        if len(c) == 0:
            return [], False
        s = self.key_scores(v, c)
        order = np.lexsort((c, -s.astype(np.float64)))
        c, s = c[order], s[order]
        P = pair_scores(self.metric, self.table, self.k, self.codes[c], self.codes[c])
        return prune_select(s, c, P, self.degree, self.alpha), False


def upper_levels(oracle, codes, codebooks, k, dim, centroid, table, metric, members, **kw):
    """every upper level built by the model over its members' code rows: [(ids, adj in global ids)]"""
    out = []
    for ids in members:
        if len(ids) > 1:
            sub, _ = PQBuildModel(oracle, codes[ids], codebooks, k, dim, centroid, table, metric, **kw).build()
            adj = np.where(sub >= 0, ids[np.clip(sub, 0, None)], -1).astype(np.int32)
        else:
            adj = np.full((len(ids), kw["M"]), -1, np.int32)
        out.append((ids, adj))
    return out
