"""The device graph build over BQ codes and its maintenance (jv_graph_build_bq, jv_graph_add_nodes_bq, jv_graph_remove_deleted_bq:
build.cu prune_kernel<.., KIND_BQ>) restated on the host, as the checker of jv_builder_create_bq / jv_builder_create_from_graph_bq
+ jv_builder_* and of the removal.

It is build_model.BuildModel with the scores of BuildScoreProvider.bqBuildScoreProvider:
  query   : c_v as fp32, +1 where bit j is set and -1 where it is clear (bq_decode_kernel); the walk re-encodes it to c_v exactly
  search  : the oracle's traversal (jvo_graph_search) with jvo_scorer_bq over that query: 1 - hd / dim, no rerank,
            topK = rerankK = beam
  keys    : the same scorer's score of every candidate
  pairs   : jvo_bq_score(c_a, c_b) = 1 - hd(c_a, c_b) / dim
  prune   : pq_build_model.prune_select (prune_kernel's selection restated literally)
No score depends on the metric. Hamming distances are exact integers mapped by one correctly rounded divide and subtract, so every
score is the device's own bits in any order: nothing is flagged, and any difference from the device is a bug.

  SeededBQBuildModel : BQBuildModel started from a graph as add_model.SeededBuildModel starts BuildModel (rows with their -1 slots
                       squeezed out, inserts from the graph's entry or the first new row, insert searches that may pick only accepted rows)
  extend_levels      : add_model.extend_levels over word rows
  BQRepairModel      : delete_model.remove_deleted with the BQ prune in place of retain_diverse"""
import ctypes as C

import numpy as np

import add_model as am
import build_model as bm
import delete_model as dm
import oracle_lib as o
import pq_build_model as pm
from oracle_lib import fp, ip

F32 = np.float32
U64P = C.POINTER(C.c_uint64)

# the capacities of the removal's BQ prune (build.cu CODE_REPAIR_TIER_MAX): a row runs at the smallest that holds its candidates
REPAIR_TIERS = (64, 128, 256, 1024, 2048, 8192)


def repair_tier(ncand):
    return next(t for t, cap in enumerate(REPAIR_TIERS) if ncand <= cap or cap == REPAIR_TIERS[-1])


def wp(a):
    return a.ctypes.data_as(U64P)


def decode(words, dim):
    """bq_decode_kernel for every row of words [n][W]: float32 [n][dim], +1 where bit j is set, -1 where it is clear"""
    bits = (words[:, :, None] >> np.arange(64, dtype=np.uint64)[None, None, :]) & np.uint64(1)
    bits = bits.reshape(words.shape[0], -1)[:, :dim]
    return np.where(bits == 1, F32(1), F32(-1)).astype(F32)


def popcount64(x):
    """per-element population count of a uint64 array"""
    x = x.astype(np.uint64)
    return np.unpackbits(x.view(np.uint8).reshape(x.shape + (8,)), axis=-1).sum(-1).astype(np.int64)


def pair_scores(words, dim, a, b):
    """BQVectors.similarityBetween for word rows a [na] against b [nb] (ids): float32 [na][nb], 1 - hd / dim in float32"""
    hd = popcount64(words[a][:, None, :] ^ words[b][None, :, :]).sum(-1)
    return (F32(1) - (hd.astype(F32) / F32(dim))).astype(F32)


class _PairColumns:
    """what prune_select reads of the pair matrix, P[live, pick], computed when asked"""

    def __init__(self, words, dim, ids):
        self.words, self.dim, self.ids = words, dim, ids

    def __getitem__(self, key):
        live, pick = key
        return pair_scores(self.words, self.dim, self.ids[live], self.ids[pick:pick + 1])[:, 0]


class BQBuildModel(bm.BuildModel):
    def __init__(self, oracle, words, dim, metric, M, beam, **kw):
        self.words = np.ascontiguousarray(words, np.uint64)
        self.queries = decode(self.words, dim)
        super().__init__(oracle, self.queries, metric, M, beam, **kw)

    def scorer(self, v):
        """the BQ scorer of v's query (the caller frees it)"""
        return self.L.jvo_scorer_bq(wp(self.words), self.n, self.dim, fp(self.queries[v]))

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
        return pm.prune_select(s, c, _PairColumns(self.words, self.dim, c), self.degree, self.alpha), False


def upper_levels(oracle, words, dim, metric, members, **kw):
    """every upper level built by the model over its members' word rows: [(ids, adj in global ids)]"""
    out = []
    for ids in members:
        if len(ids) > 1:
            sub, _ = BQBuildModel(oracle, words[ids], dim, metric, **kw).build()
            adj = np.where(sub >= 0, ids[np.clip(sub, 0, None)], -1).astype(np.int32)
        else:
            adj = np.full((len(ids), kw["M"]), -1, np.int32)
        out.append((ids, adj))
    return out


class SeededBQBuildModel(BQBuildModel):
    def __init__(self, oracle, words, dim, metric, rows, entry, accept=None, **kw):
        """rows [n0][w] of row ids (-1 = empty slot); entry < 0: row n0 becomes the entry; accept: bool [n] of the rows an insert
        may pick as neighbours (None = all)"""
        super().__init__(oracle, words, dim, metric, **kw)
        rows = np.asarray(rows, np.int32)
        n0 = rows.shape[0]
        for v in range(n0):
            valid = rows[v][rows[v] >= 0]
            self.adj[v, :len(valid)] = valid
            self.deg[v] = len(valid)
        self.entry = entry if entry >= 0 else n0
        self.inserted = min(self.n, n0 if entry >= 0 else n0 + 1)
        self.accept = am.pack_bits(accept) if accept is not None else None

    def search(self, u):
        g = o.make_graph(self.adj, self.entry)
        sf = self.scorer(u)
        nodes = np.full(self.beam, -1, np.int32)
        scores = np.zeros(self.beam, F32)
        acc = self.accept.ctypes.data_as(C.POINTER(C.c_uint32)) if self.accept is not None else None
        cnt = self.L.jvo_graph_search_ex(C.byref(g), sf, None, self.beam, self.beam, 0.0, 0.0, acc, ip(nodes), fp(scores), None)
        self.L.jvo_scorer_free(sf)
        return [int(x) for x in nodes[:cnt] if x >= 0]


def extend_levels(oracle, words, dim, metric, levels, entry, n0, seed, marks=None, **kw):
    """the levels [(ids, adj in node ids)] of a graph of n0 nodes after rows [n0, len(words)) were added; marks: bool [n0] of marked
    nodes. Returns ([(ids, adj)], entry)"""
    fresh = am.added_levels(n0, len(words), kw["M"], seed)
    out = []
    for lv in range(1, max(len(levels), len(fresh)) + 1):
        new = fresh[lv - 1] if lv <= len(fresh) else np.zeros(0, np.int32)
        if lv > len(levels):
            out += upper_levels(oracle, words, dim, metric, [new], **kw)
            continue
        ids, adj = levels[lv - 1]
        if len(new) == 0:
            out.append((ids, adj))
            continue
        allids = np.concatenate([ids, new]).astype(np.int32)
        row = {int(v): r for r, v in enumerate(ids)}
        local = np.array([[row.get(int(x), -1) if x >= 0 else -1 for x in r] for r in adj], np.int32).reshape(len(ids), -1)
        accept = None if marks is None else np.array([r >= len(ids) or not marks[v] for r, v in enumerate(allids)])
        sub, _ = SeededBQBuildModel(oracle, words[allids], dim, metric, local, row.get(int(entry), 0), accept, **kw).build()
        out.append((allids, np.where(sub >= 0, allids[np.clip(sub, 0, None)], -1).astype(np.int32)))
    if len(fresh) > len(levels):
        entry = int(out[-1][0][0])
    return out, entry


class BQRepairModel(BQBuildModel):
    def __init__(self, oracle, words, dim, metric, degree, alpha=1.2):
        super().__init__(oracle, words, dim, metric, M=degree, beam=1, alpha=alpha)

    def remove_deleted(self, adj0, entry, upper, deleted, seed=0, holes=None):
        """delete_model.remove_deleted's result with every repaired row pruned by the BQ prune"""
        saved = dm.retain_diverse
        dm.retain_diverse = lambda metric, data, v, cands, degree, alpha, key_scores=None: self.prune(v, cands)
        try:
            return dm.remove_deleted(self.queries, self.metric, adj0, entry, upper, deleted, alpha=self.alpha, seed=seed, holes=holes)
        finally:
            dm.retain_diverse = saved
