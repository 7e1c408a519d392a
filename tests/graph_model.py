"""The device graph build, add and removal (build.cu build_graph_flat, api.cu) restated on the host, batch by batch, as the checker
of jv_builder_*, over any of the three score providers.

The mirror holds what the device holds: the level-0 adjacency [n][row_cap] (-1 padded) and deg[n]. Each step is restated
literally, so every row the builder writes has one value to compare against:
  insert   : for every node u of the batch, the oracle's warp-order traversal (jvo_graph_search_ex from the entry, rows row_cap
             wide, topK = rerankK = beam, only accepted rows picked) of the mirror graph with the provider's scorer of u's query;
             candidates = its results + the in-progress window (prune_candidate); then the provider's robust prune
  apply    : the rows are written, then the back-link pairs (t, u), skipping a pair whose ends are both in the batch and already
             name each other, sorted by (target, source); pair i of t's segment lands at deg_before[t] + rank, or is dropped (and
             counted) at or past row_cap; a target whose new degree passes hard_max = (int)(overflow * M) joins the re-prune list
  re-prune : each listed row is pruned over its own entries
  cleanup  : the rows longer than M are re-pruned, then every row is cut to min(deg, M)
A build starts from node 0 with an empty row. An add (jv_graph_add_nodes*, jv_builder_create_from_graph*) starts from the graph's
rows, each with its -1 slots squeezed out (entries keep their order), inserts from the graph's entry (no entry: the first new row,
as node 0 is for a build), and its insert searches may only pick accepted rows: marked nodes are walked through but never become a
neighbour. Levels: api.cu assign_levels / add_upper_levels restated, every upper level a build over its members' rows.

The score providers (BuildScoreProvider):
  F32Scores : fp32 rows. The query is the row; the prune is delete_model.retain_diverse over the device's own key bits
              (jvo_compare_f32_warp). A row is flagged when one of its prune decisions is a near tie under delete_model.pair_bound;
              only flagged rows may differ from the device.
  PQScores  : pqBuildScoreProvider. The query is decode(c_v) (per sub-space the codebook row plus the global centroid, one fp32 add
              per element); the scorer is jvo_scorer_pq over it in the kernels' order (the walk's own bits, no rerank); keys are the
              same scorer's scores; pairs are pair_pq_table (scorers.cuh) restated in float32 over a given centroid-pair table
              (lane l sums the entries of sub-spaces m = l, l + 32, ... in increasing m, then the xor butterfly 16, 8, 4, 2, 1; cosine
              sum / sqrt(n1 n2); the score map last).
  BQScores  : bqBuildScoreProvider. The query is c_v as fp32, +1 where bit j is set and -1 where it is clear (bq_decode_kernel); the
              walk re-encodes it to c_v exactly; the scorer is jvo_scorer_bq (1 - hd / dim, no rerank); pairs are 1 - hd(c_a, c_b) /
              dim. No score depends on the metric.
For PQ and BQ the prune is prune_kernel's selection restated literally (prune_select) over the candidates in key order. Every score
is then the device's own bits (Hamming distances are exact integers mapped by one correctly rounded divide and subtract), so nothing
is flagged: any difference from the device is a bug."""
import ctypes as C
import math

import numpy as np

import delete_model as dm
import oracle_lib as o
from oracle_lib import bp, fp, ip

F32 = np.float32
U64P = C.POINTER(C.c_uint64)
_M64 = (1 << 64) - 1


# ------------------------------------------------------------------------------------------------ PQ scores
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


# ------------------------------------------------------------------------------------------------ BQ scores
def wp(a):
    return a.ctypes.data_as(U64P)


def bq_decode(words, dim):
    """bq_decode_kernel for every row of words [n][W]: float32 [n][dim], +1 where bit j is set, -1 where it is clear"""
    bits = (words[:, :, None] >> np.arange(64, dtype=np.uint64)[None, None, :]) & np.uint64(1)
    bits = bits.reshape(words.shape[0], -1)[:, :dim]
    return np.where(bits == 1, F32(1), F32(-1)).astype(F32)


def popcount64(x):
    """per-element population count of a uint64 array"""
    x = x.astype(np.uint64)
    return np.unpackbits(x.view(np.uint8).reshape(x.shape + (8,)), axis=-1).sum(-1).astype(np.int64)


def bq_pair_scores(words, dim, a, b):
    """BQVectors.similarityBetween for word rows a [na] against b [nb] (ids): float32 [na][nb], 1 - hd / dim in float32"""
    hd = popcount64(words[a][:, None, :] ^ words[b][None, :, :]).sum(-1)
    return (F32(1) - (hd.astype(F32) / F32(dim))).astype(F32)


# ------------------------------------------------------------------------------------------------ the prune over codes
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


class _PairColumns:
    """what prune_select reads of the pair matrix, P[live, pick], computed when asked: a row of thousands of candidates folds at most
    `degree` columns, never the whole matrix"""

    def __init__(self, scores, ids):
        self.scores, self.ids = scores, ids

    def __getitem__(self, key):
        live, pick = key
        return self.scores.pairs(self.ids[live], self.ids[pick:pick + 1])[:, 0]


class _CodeScores:
    """what the PQ and BQ providers share: keys from the walk's own scorer, and prune_kernel's selection over them"""

    def key_scores(self, v, ids):
        sf = self.scorer(v)
        out = np.array([self.L.jvo_scorer_score(sf, int(i)) for i in ids], F32)
        self.L.jvo_scorer_free(sf)
        return out

    def prune(self, v, cands, degree, alpha):
        c = np.array(sorted(set(int(x) for x in cands) - {int(v)}), dtype=np.int64)
        if len(c) == 0:
            return [], False
        s = self.key_scores(v, c)
        order = np.lexsort((c, -s.astype(np.float64)))
        c, s = c[order], s[order]
        return prune_select(s, c, _PairColumns(self, c), degree, alpha), False


# ------------------------------------------------------------------------------------------------ score providers
class F32Scores:
    def __init__(self, oracle, data, metric):
        self.L, self.metric = oracle, metric
        self.queries = np.ascontiguousarray(data, dtype=F32)
        self.n, self.dim = self.queries.shape

    def scorer(self, v):
        """the warp-order fp32 scorer of row v (the caller frees it)"""
        sf = self.L.jvo_scorer_f32(self.metric, fp(self.queries), self.n, self.dim, fp(self.queries[v]))
        self.L.jvo_scorer_set_order(sf, 1)
        return sf

    def key_scores(self, v, ids):
        d, m, L = self.queries, self.metric, self.L
        return np.array([L.jvo_compare_f32_warp(m, fp(d[v]), fp(d[i]), self.dim) for i in ids], F32)

    def prune(self, v, cands, degree, alpha):
        return dm.retain_diverse(self.metric, self.queries, v, cands, degree, alpha, self.key_scores)

    def subset(self, ids):
        return F32Scores(self.L, self.queries[ids], self.metric)


class PQScores(_CodeScores):
    def __init__(self, oracle, codes, codebooks, k, dim, centroid, table, metric):
        self.L, self.metric = oracle, metric
        self.codes = np.ascontiguousarray(codes, np.uint8)
        self.codebooks = np.ascontiguousarray(codebooks, F32).reshape(-1)
        self.k, self.dim, self.pq_m = k, dim, self.codes.shape[1]
        self.centroid = None if centroid is None else np.ascontiguousarray(centroid, F32)
        self.table = np.ascontiguousarray(table, F32)
        self.queries = decode(self.codes, self.codebooks, *o.pq_layout(dim, self.pq_m), k, self.centroid)
        self.n = len(self.codes)

    def scorer(self, v):
        """the warp-order PQ scorer of decode(c_v) (the caller frees it)"""
        sf = self.L.jvo_scorer_pq(self.metric, fp(self.codebooks), self.pq_m, self.k, self.dim, fp(self.centroid), bp(self.codes), self.n,
                                  fp(self.queries[v]))
        self.L.jvo_scorer_set_order(sf, 1)
        return sf

    def pairs(self, a, b):
        return pair_scores(self.metric, self.table, self.k, self.codes[a], self.codes[b])

    def subset(self, ids):
        return PQScores(self.L, self.codes[ids], self.codebooks, self.k, self.dim, self.centroid, self.table, self.metric)


class BQScores(_CodeScores):
    def __init__(self, oracle, words, dim, metric):
        self.L, self.metric, self.dim = oracle, metric, dim
        self.words = np.ascontiguousarray(words, np.uint64)
        self.queries = bq_decode(self.words, dim)
        self.n = len(self.words)

    def scorer(self, v):
        """the BQ scorer of v's query (the caller frees it)"""
        return self.L.jvo_scorer_bq(wp(self.words), self.n, self.dim, fp(self.queries[v]))

    def pairs(self, a, b):
        return bq_pair_scores(self.words, self.dim, a, b)

    def subset(self, ids):
        return BQScores(self.L, self.words[ids], self.dim, self.metric)


# ------------------------------------------------------------------------------------------------ the builder
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


def pack_bits(mask):
    """bool [n] -> uint32 words, bit (i & 31) of word (i >> 5)"""
    m = np.asarray(mask, bool)
    m = np.concatenate([m, np.zeros((-len(m)) % 32, bool)])
    return np.ascontiguousarray(np.packbits(m, bitorder="little").view(np.uint32))


class BuildModel:
    def __init__(self, scores, M, beam, overflow=1.2, alpha=1.2, max_batch=0, window=-1, batch_div=32, rows=None, entry=-1, accept=None):
        """a build over scores' rows, or with rows [n0][w] of row ids (-1 = empty slot) an add of rows [n0, n) to that graph.
        entry < 0: row n0 becomes the entry; accept: bool [n] of the rows an insert may pick as neighbours (None = all)"""
        self.scores, self.L = scores, scores.L
        self.n = scores.n
        self.degree, self.beam, self.alpha = M, beam, alpha
        self.hard_max = int(np.float32(overflow) * np.float32(M))
        self.row_cap = max(2 * M, self.hard_max + 1)
        self.max_batch = max_batch if max_batch > 0 else 16384
        self.window = window if window >= 0 else default_window(beam)
        self.batch_div = batch_div
        self.adj = np.full((self.n, self.row_cap), -1, np.int32)
        self.deg = np.zeros(self.n, np.int64)
        rows = np.zeros((0, M), np.int32) if rows is None else np.asarray(rows, np.int32)
        n0 = rows.shape[0]
        for v in range(n0):
            valid = rows[v][rows[v] >= 0]
            self.adj[v, :len(valid)] = valid
            self.deg[v] = len(valid)
        self.entry = entry if entry >= 0 else n0
        self.inserted = min(self.n, n0 if entry >= 0 else n0 + 1)
        self.accept = pack_bits(accept) if accept is not None else None
        self.dropped = 0
        self.flagged = 0
        self.prunes = 0

    def prune(self, v, cands):
        sel, flag = self.scores.prune(v, cands, self.degree, self.alpha)
        self.flagged += int(flag)
        self.prunes += 1
        return sel, flag

    def next_batch(self):
        if self.inserted >= self.n:
            return None
        b = min(max(1, self.inserted // self.batch_div), self.max_batch, self.n - self.inserted)
        return self.inserted, b

    def search(self, u):
        g = o.make_graph(self.adj, self.entry)
        sf = self.scores.scorer(u)
        nodes = np.full(self.beam, -1, np.int32)
        scores = np.zeros(self.beam, F32)
        acc = self.accept.ctypes.data_as(C.POINTER(C.c_uint32)) if self.accept is not None else None
        cnt = self.L.jvo_graph_search_ex(C.byref(g), sf, None, self.beam, self.beam, 0.0, 0.0, acc, ip(nodes), fp(scores), None)
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


# ------------------------------------------------------------------------------------------------ levels
def level_draws(n, degree, seed):
    """api.cu draw_levels: level(node i) = floor(-ln U_i / ln M), U_i the i-th draw of xorshift64"""
    st = seed if seed else 0x9E3779B97F4A7C15
    ml = 1.0 if degree == 1 else 1.0 / math.log(degree)
    level = np.empty(n, np.int64)
    for i in range(n):
        st ^= (st << 13) & _M64
        st ^= st >> 7
        st ^= (st << 17) & _M64
        u = ((st >> 11) + 1) * (1.0 / 9007199254740993.0)
        level[i] = int(-math.log(u) * ml)
    return level


def assign_levels(n, degree, seed):
    """api.cu assign_levels: (members of levels 1.., entry node = the first node of the top level)"""
    level = level_draws(n, degree, seed)
    maxl = int(level.max()) if n else 0
    entry = int(np.flatnonzero(level == maxl)[0]) if n else 0
    return [np.flatnonzero(level >= lv).astype(np.int32) for lv in range(1, maxl + 1)], entry


def added_levels(n0, n, degree, seed):
    """the upper levels new nodes [n0, n) join: node i takes draw i of level_draws(n); the new members of levels 1.., ascending"""
    level = level_draws(n, degree, seed)[n0:]
    top = int(level.max()) if len(level) else 0
    return [(n0 + np.flatnonzero(level >= lv)).astype(np.int32) for lv in range(1, top + 1)]


def _level(scores, ids, **kw):
    """a level over the rows ids (seeded by kw's rows when given): (ids, adj in global ids, flagged prunes)"""
    sub, flagged = BuildModel(scores.subset(ids), **kw).build()
    return ids, np.where(sub >= 0, ids[np.clip(sub, 0, None)], -1).astype(np.int32), flagged


def upper_levels(scores, members, **kw):
    """every upper level built by the model over its members' rows: [(ids, adj in global ids, flagged prunes)]"""
    return [_level(scores, ids, **kw) if len(ids) > 1 else (ids, np.full((len(ids), kw["M"]), -1, np.int32), 0) for ids in members]


def extend_levels(scores, levels, entry, n0, seed, marks=None, **kw):
    """api.cu add_upper_levels: the levels [(ids, adj in node ids)] of a graph of n0 nodes after rows [n0, scores.n) were added; a level
    that gains members is a seeded build over its old members then its new ones, from the entry's row; a level above the top is built
    over its new members and its lowest id becomes the entry. marks: bool [n0] of marked nodes.
    Returns ([(ids, adj, flagged prunes)], entry)"""
    fresh = added_levels(n0, scores.n, kw["M"], seed)
    out = []
    for lv in range(1, max(len(levels), len(fresh)) + 1):
        new = fresh[lv - 1] if lv <= len(fresh) else np.zeros(0, np.int32)
        if lv > len(levels):
            out += upper_levels(scores, [new], **kw)
            continue
        ids, adj = levels[lv - 1]
        if len(new) == 0:
            out.append((ids, adj, 0))
            continue
        allids = np.concatenate([ids, new]).astype(np.int32)
        row = {int(v): r for r, v in enumerate(ids)}
        local = np.array([[row.get(int(x), -1) if x >= 0 else -1 for x in r] for r in adj], np.int32).reshape(len(ids), -1)
        accept = None if marks is None else np.array([r >= len(ids) or not marks[v] for r, v in enumerate(allids)])
        out.append(_level(scores, allids, rows=local, entry=row.get(int(entry), 0), accept=accept, **kw))
    if len(fresh) > len(levels):
        entry = int(out[-1][0][0])
    return out, entry
