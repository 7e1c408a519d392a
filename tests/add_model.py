"""An add into an existing graph (jv_graph_add_nodes, jv_builder_create_from_graph) restated on the host: the build's model
(tests/build_model.py) started from the graph instead of from node 0.

  SeededBuildModel : BuildModel whose first rows are the graph's, each with its -1 slots squeezed out (entries keep their order),
                     whose inserts start at the graph's entry (no entry: the first new row, with an empty row, as node 0 is for a
                     build) and whose insert searches (jvo_graph_search_ex) may only pick the accepted rows: marked nodes are walked
                     through but never become a neighbour
  level_draws      : api.cu draw_levels, the build's level of node i
  added_levels     : the upper levels the new nodes join (draw i for node i of n)
  extend_levels    : api.cu add_upper_levels: a level that gains members is a seeded build over its old members then its new ones,
                     from the entry's row; a level above the top is built over its new members and its lowest id becomes the entry"""
import ctypes as C
import math

import numpy as np

import build_model as bm
import oracle_lib as o
from oracle_lib import fp, ip

_M64 = (1 << 64) - 1


def pack_bits(mask):
    """bool [n] -> uint32 words, bit (i & 31) of word (i >> 5)"""
    m = np.asarray(mask, bool)
    m = np.concatenate([m, np.zeros((-len(m)) % 32, bool)])
    return np.ascontiguousarray(np.packbits(m, bitorder="little").view(np.uint32))


class SeededBuildModel(bm.BuildModel):
    def __init__(self, oracle, data, metric, rows, entry, accept=None, **kw):
        """rows [n0][w] of row ids (-1 = empty slot); entry < 0: row n0 becomes the entry; accept: bool [n] of the rows an insert
        may pick as neighbours (None = all)"""
        super().__init__(oracle, data, metric, **kw)
        rows = np.asarray(rows, np.int32)
        n0 = rows.shape[0]
        for v in range(n0):
            valid = rows[v][rows[v] >= 0]
            self.adj[v, :len(valid)] = valid
            self.deg[v] = len(valid)
        self.entry = entry if entry >= 0 else n0
        self.inserted = min(self.n, n0 if entry >= 0 else n0 + 1)
        self.accept = pack_bits(accept) if accept is not None else None

    def search(self, u):
        g = o.make_graph(self.adj, self.entry)
        sf = self.L.jvo_scorer_f32(self.metric, fp(self.data), self.n, self.dim, fp(self.data[u]))
        self.L.jvo_scorer_set_order(sf, 1)
        nodes = np.full(self.beam, -1, np.int32)
        scores = np.zeros(self.beam, np.float32)
        acc = self.accept.ctypes.data_as(C.POINTER(C.c_uint32)) if self.accept is not None else None
        cnt = self.L.jvo_graph_search_ex(C.byref(g), sf, None, self.beam, self.beam, 0.0, 0.0, acc, ip(nodes), fp(scores), None)
        self.L.jvo_scorer_free(sf)
        return [int(x) for x in nodes[:cnt] if x >= 0]


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


def added_levels(n0, n, degree, seed):
    """the upper levels new nodes [n0, n) join: node i takes draw i of level_draws(n); the new members of levels 1.., ascending"""
    level = level_draws(n, degree, seed)[n0:]
    top = int(level.max()) if len(level) else 0
    return [(n0 + np.flatnonzero(level >= lv)).astype(np.int32) for lv in range(1, top + 1)]


def extend_levels(oracle, data, metric, levels, entry, n0, seed, marks=None, **kw):
    """the levels [(ids, adj in node ids)] of a graph of n0 nodes after nodes [n0, len(data)) were added; marks: bool [n0] of marked
    nodes. Returns ([(ids, adj, flagged prunes)], entry)"""
    fresh = added_levels(n0, len(data), kw["M"], seed)
    out = []
    for lv in range(1, max(len(levels), len(fresh)) + 1):
        new = fresh[lv - 1] if lv <= len(fresh) else np.zeros(0, np.int32)
        if lv > len(levels):
            out += bm.upper_levels(oracle, data, metric, [new], **kw)
            continue
        ids, adj = levels[lv - 1]
        if len(new) == 0:
            out.append((ids, adj, 0))
            continue
        allids = np.concatenate([ids, new]).astype(np.int32)
        row = {int(v): r for r, v in enumerate(ids)}
        local = np.array([[row.get(int(x), -1) if x >= 0 else -1 for x in r] for r in adj], np.int32).reshape(len(ids), -1)
        accept = None if marks is None else np.array([r >= len(ids) or not marks[v] for r, v in enumerate(allids)])
        sub, flagged = SeededBuildModel(oracle, data[allids], metric, local, row.get(int(entry), 0), accept, **kw).build()
        out.append((allids, np.where(sub >= 0, allids[np.clip(sub, 0, None)], -1).astype(np.int32), flagged))
    if len(fresh) > len(levels):
        entry = int(out[-1][0][0])
    return out, entry
