"""The device graph build (build.cu build_graph_flat) restated on the host, batch by batch, as the checker of jv_builder_*.

The mirror holds what the device holds: the level-0 adjacency [n][row_cap] (-1 padded) and deg[n]. Each step is restated
literally, so every row the builder writes has one value to compare against:
  insert   : for every node u of the batch, the oracle's warp-order traversal (jvo_graph_search, entry 0, rows row_cap wide,
             topK = rerankK = beam) of the mirror graph; candidates = its results + the in-progress window (prune_candidate); the
             robust prune is delete_model.retain_diverse over the device's own key bits (jvo_compare_f32_warp)
  apply    : the rows are written, then the back-link pairs (t, u), skipping a pair whose ends are both in the batch and already
             name each other, sorted by (target, source); pair i of t's segment lands at deg_before[t] + rank, or is dropped (and
             counted) at or past row_cap; a target whose new degree passes hard_max = (int)(overflow * M) joins the re-prune list
  re-prune : each listed row is pruned over its own entries
  cleanup  : the rows longer than M are re-pruned, then every row is cut to min(deg, M)
A row is flagged when one of its prune decisions is a near tie under delete_model.pair_bound; only flagged rows may differ from
the device. Levels: assign_levels (api.cu) restated, every upper level a build over its members' rows."""
import ctypes as C
import math

import numpy as np

import delete_model as dm
import oracle_lib as o
from oracle_lib import fp, ip

_M64 = (1 << 64) - 1


def default_window(beam):
    """the in-progress window when none is given: what still fits the 128-candidate Gram tile next to the beam, at most 32"""
    return max(0, min(32, 128 - beam))


def window_candidates(u, window, first, count):
    """prune_candidate's window part: the W batch nodes around u in insertion order, u itself skipped"""
    out = []
    half = window >> 1
    for j in range(window):
        w = u - half + j
        if w >= u:
            w += 1
        if first <= w < first + count:
            out.append(w)
    return out


class BuildModel:
    def __init__(self, oracle, data, metric, M, beam, overflow=1.2, alpha=1.2, max_batch=0, window=-1, batch_div=32):
        self.L = oracle
        self.data = np.ascontiguousarray(data, dtype=np.float32)
        self.n, self.dim = self.data.shape
        self.metric, self.degree, self.beam, self.alpha = metric, M, beam, alpha
        self.hard_max = int(np.float32(overflow) * np.float32(M))
        self.row_cap = max(2 * M, self.hard_max + 1)
        self.max_batch = max_batch if max_batch > 0 else 16384
        self.window = window if window >= 0 else default_window(beam)
        self.batch_div = batch_div
        self.adj = np.full((self.n, self.row_cap), -1, np.int32)
        self.deg = np.zeros(self.n, np.int64)
        self.inserted = 1
        self.dropped = 0
        self.flagged = 0
        self.prunes = 0

    def key_scores(self, v, ids):
        d, m, L = self.data, self.metric, self.L
        return np.array([L.jvo_compare_f32_warp(m, fp(d[v]), fp(d[i]), self.dim) for i in ids], np.float32)

    def prune(self, v, cands):
        sel, flag = dm.retain_diverse(self.metric, self.data, v, cands, self.degree, self.alpha, self.key_scores)
        self.flagged += int(flag)
        self.prunes += 1
        return sel, flag

    def next_batch(self):
        if self.inserted >= self.n:
            return None
        b = min(max(1, self.inserted // self.batch_div), self.max_batch, self.n - self.inserted)
        return self.inserted, b

    def search(self, u):
        g = o.make_graph(self.adj, 0)
        sf = self.L.jvo_scorer_f32(self.metric, fp(self.data), self.n, self.dim, fp(self.data[u]))
        self.L.jvo_scorer_set_order(sf, 1)
        nodes = np.full(self.beam, -1, np.int32)
        scores = np.zeros(self.beam, np.float32)
        cnt = self.L.jvo_graph_search(C.byref(g), sf, None, self.beam, self.beam, ip(nodes), fp(scores), None)
        self.L.jvo_scorer_free(sf)
        return [int(x) for x in nodes[:cnt] if x >= 0]

    def insert_rows(self, first, count):
        """the batch's new rows [count][M] (-1 padded), their degrees and near-tie flags; the mirror is not changed"""
        rows = np.full((count, self.degree), -1, np.int32)
        rdeg = np.zeros(count, np.int32)
        flags = np.zeros(count, bool)
        for i in range(count):
            u = first + i
            cands = self.search(u) + window_candidates(u, self.window, first, count)
            sel, flags[i] = self.prune(u, cands)
            rows[i, :len(sel)] = sel
            rdeg[i] = len(sel)
        return rows, rdeg, flags

    def apply_new(self, first, count, rows, rdeg):
        """writes the rows and their back-links; returns the sorted list of rows that passed hard_max"""
        self.adj[first:first + count] = -1
        self.adj[first:first + count, :self.degree] = rows
        self.deg[first:first + count] = rdeg
        pairs = []
        for i in range(count):
            u = first + i
            for t in rows[i]:
                t = int(t)
                if t < 0:
                    continue
                if first <= t < first + count and u in rows[t - first]:
                    continue  # t chose u itself in this batch: u is in t's row already
                pairs.append((t, u))
        pairs.sort()
        over = []
        k = 0
        while k < len(pairs):
            t = pairs[k][0]
            e = k
            while e < len(pairs) and pairs[e][0] == t:
                e += 1
            d0 = int(self.deg[t])
            for r in range(e - k):
                if d0 + r < self.row_cap:
                    self.adj[t, d0 + r] = pairs[k + r][1]
                else:
                    self.dropped += 1
            nd = min(self.row_cap, d0 + e - k)
            self.deg[t] = nd
            if nd > self.hard_max:
                over.append(t)
            k = e
        self.inserted = first + count
        return over

    def reprune_rows(self, lst):
        """rows [len][row_cap] pruned over their own entries, degrees and flags; the mirror is not changed"""
        rows = np.full((len(lst), self.row_cap), -1, np.int32)
        rdeg = np.zeros(len(lst), np.int32)
        flags = np.zeros(len(lst), bool)
        for i, v in enumerate(lst):
            own = [int(x) for x in self.adj[v, :min(int(self.deg[v]), self.row_cap)]]
            sel, flags[i] = self.prune(v, own)
            rows[i, :len(sel)] = sel
            rdeg[i] = len(sel)
        return rows, rdeg, flags

    def apply_repruned(self, lst, rows, rdeg):
        for i, v in enumerate(lst):
            self.adj[v] = rows[i]
            self.deg[v] = rdeg[i]

    def over_degree(self):
        return [int(v) for v in np.flatnonzero(self.deg > self.degree)]

    def compact(self):
        out = np.full((self.n, self.degree), -1, np.int32)
        for v in range(self.n):
            d = min(int(self.deg[v]), self.degree)
            out[v, :d] = self.adj[v, :d]
        return out

    def build(self):
        """the whole flat build, every step from the mirror's own rows: (adjacency [n][M], flagged prunes)"""
        while True:
            nb = self.next_batch()
            if nb is None:
                break
            first, count = nb
            rows, rdeg, _ = self.insert_rows(first, count)
            lst = self.apply_new(first, count, rows, rdeg)
            self.apply_repruned(lst, *self.reprune_rows(lst)[:2])
        lst = self.over_degree()
        self.apply_repruned(lst, *self.reprune_rows(lst)[:2])
        return self.compact(), self.flagged


def assign_levels(n, degree, seed):
    """api.cu assign_levels: level(node) = floor(-ln U / ln M), U from xorshift64; (members of levels 1.., entry node)"""
    st = seed if seed else 0x9E3779B97F4A7C15
    ml = 1.0 if degree == 1 else 1.0 / math.log(degree)
    level = np.empty(n, np.int64)
    for i in range(n):
        st ^= (st << 13) & _M64
        st ^= st >> 7
        st ^= (st << 17) & _M64
        u = ((st >> 11) + 1) * (1.0 / 9007199254740993.0)
        level[i] = int(-math.log(u) * ml)
    maxl = int(level.max()) if n else 0
    entry = int(np.flatnonzero(level == maxl)[0]) if n else 0
    return [np.flatnonzero(level >= lv).astype(np.int32) for lv in range(1, maxl + 1)], entry


def upper_levels(oracle, data, metric, members, **kw):
    """every upper level built by the model over its members' rows: [(ids, adj in global ids, flagged prunes)]"""
    out = []
    for ids in members:
        if len(ids) > 1:
            sub, flagged = BuildModel(oracle, data[ids], metric, **kw).build()
            adj = np.where(sub >= 0, ids[np.clip(sub, 0, None)], -1).astype(np.int32)
        else:
            adj, flagged = np.full((len(ids), kw["M"]), -1, np.int32), 0
        out.append((ids, adj, flagged))
    return out
