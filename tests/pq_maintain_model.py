"""Adds to and removals from a graph over PQ codes (jv_graph_add_nodes_pq, jv_builder_create_from_graph_pq, jv_graph_remove_deleted_pq)
restated on the host.

  SeededPQBuildModel : pq_build_model.PQBuildModel started from a graph the way add_model.SeededBuildModel starts BuildModel: the
                       graph's rows with their -1 slots squeezed out, the inserts from the graph's entry (no entry: the first new
                       row), and insert searches (jvo_graph_search_ex over the PQ scorer of decode(c_u)) that may only pick accepted rows
  extend_levels      : add_model.extend_levels over code rows: a level that gains members is a seeded PQ build over its old members'
                       codes then its new ones
  PQRepairModel      : delete_model.remove_deleted — its candidate gathering, random fallback (repair_random) and entry rule — with
                       the PQ prune in place of retain_diverse: keys from PQBuildModel.key_scores (the walk's ADC bits under
                       decode(c_v)'s LUT), selection by pq_build_model.prune_select over pair_scores (pair_pq_table's warp order)
Every score is the device's own bits, so no row is ever flagged: any difference from the device is a bug."""
import ctypes as C

import numpy as np

import add_model as am
import delete_model as dm
import oracle_lib as o
import pq_build_model as pm
from oracle_lib import fp, ip

# the capacities of the removal's PQ prune (build.cu PQ_REPAIR_TIER_MAX): a row runs at the smallest that holds its candidates
PQ_REPAIR_TIERS = (64, 128, 256, 1024, 2048, 8192)


def repair_tier(ncand):
    return next(t for t, cap in enumerate(PQ_REPAIR_TIERS) if ncand <= cap or cap == PQ_REPAIR_TIERS[-1])


class SeededPQBuildModel(pm.PQBuildModel):
    def __init__(self, oracle, codes, codebooks, k, dim, centroid, table, metric, rows, entry, accept=None, **kw):
        """rows [n0][w] of row ids (-1 = empty slot); entry < 0: row n0 becomes the entry; accept: bool [n] of the rows an insert
        may pick as neighbours (None = all)"""
        super().__init__(oracle, codes, codebooks, k, dim, centroid, table, metric, **kw)
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
        scores = np.zeros(self.beam, np.float32)
        acc = self.accept.ctypes.data_as(C.POINTER(C.c_uint32)) if self.accept is not None else None
        cnt = self.L.jvo_graph_search_ex(C.byref(g), sf, None, self.beam, self.beam, 0.0, 0.0, acc, ip(nodes), fp(scores), None)
        self.L.jvo_scorer_free(sf)
        return [int(x) for x in nodes[:cnt] if x >= 0]


def extend_levels(oracle, codes, codebooks, k, dim, centroid, table, metric, levels, entry, n0, seed, marks=None, **kw):
    """the levels [(ids, adj in node ids)] of a graph of n0 nodes after rows [n0, len(codes)) were added; marks: bool [n0] of marked
    nodes. Returns ([(ids, adj)], entry)"""
    fresh = am.added_levels(n0, len(codes), kw["M"], seed)
    out = []
    for lv in range(1, max(len(levels), len(fresh)) + 1):
        new = fresh[lv - 1] if lv <= len(fresh) else np.zeros(0, np.int32)
        if lv > len(levels):
            out += pm.upper_levels(oracle, codes, codebooks, k, dim, centroid, table, metric, [new], **kw)
            continue
        ids, adj = levels[lv - 1]
        if len(new) == 0:
            out.append((ids, adj))
            continue
        allids = np.concatenate([ids, new]).astype(np.int32)
        row = {int(v): r for r, v in enumerate(ids)}
        local = np.array([[row.get(int(x), -1) if x >= 0 else -1 for x in r] for r in adj], np.int32).reshape(len(ids), -1)
        accept = None if marks is None else np.array([r >= len(ids) or not marks[v] for r, v in enumerate(allids)])
        sub, _ = SeededPQBuildModel(oracle, codes[allids], codebooks, k, dim, centroid, table, metric, local, row.get(int(entry), 0), accept, **kw).build()
        out.append((allids, np.where(sub >= 0, allids[np.clip(sub, 0, None)], -1).astype(np.int32)))
    if len(fresh) > len(levels):
        entry = int(out[-1][0][0])
    return out, entry


class _PairColumns:
    """what prune_select reads of the pair matrix, P[live, pick], computed when asked: a row of thousands of candidates folds at most
    `degree` columns, never the whole matrix"""

    def __init__(self, metric, table, k, codes):
        self.metric, self.table, self.k, self.codes = metric, table, k, codes

    def __getitem__(self, key):
        live, pick = key
        return pm.pair_scores(self.metric, self.table, self.k, self.codes[live], self.codes[pick:pick + 1])[:, 0]


class PQRepairModel(pm.PQBuildModel):
    def __init__(self, oracle, codes, codebooks, k, dim, centroid, table, metric, degree, alpha=1.2):
        super().__init__(oracle, codes, codebooks, k, dim, centroid, table, metric, M=degree, beam=1, alpha=alpha)

    def prune(self, v, cands):
        c = np.array(sorted(set(int(x) for x in cands) - {int(v)}), dtype=np.int64)
        if len(c) == 0:
            return [], False
        s = self.key_scores(v, c)
        order = np.lexsort((c, -s.astype(np.float64)))
        c, s = c[order], s[order]
        return pm.prune_select(s, c, _PairColumns(self.metric, self.table, self.k, self.codes[c]), self.degree, self.alpha), False

    def remove_deleted(self, adj0, entry, upper, deleted, seed=0, holes=None):
        """delete_model.remove_deleted's result with every repaired row pruned by the PQ prune"""
        saved = dm.retain_diverse
        dm.retain_diverse = lambda metric, data, v, cands, degree, alpha, key_scores=None: self.prune(v, cands)
        try:
            return dm.remove_deleted(self.queries, self.metric, adj0, entry, upper, deleted, alpha=self.alpha, seed=seed, holes=holes)
        finally:
            dm.retain_diverse = saved
