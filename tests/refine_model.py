"""The refine pass (jv_graph_refine, build.cu "Refinement", DESIGN §4.3i) restated on the host, scalar and single-threaded, on
graph_model.BuildModel and its score providers (F32Scores, PQScores, BQScores).

One level at a time, the level's rows seed a BuildModel mirror (row_cap-wide rows, -1 slots squeezed out). The nodes to refine go in
ascending batches of max_batch; for each node u of a batch:
  search   : the oracle's warp-order traversal of the mirror from the level's entry, the provider's query of u, topK = rerankK = beam,
             with an accept bitset that clears u alone (what the device's exclude_ids does)
  union    : u's current row (its valid entries, in order), then the results that are not in it
  prune    : the provider's robust prune to M at alpha
Builder form (GraphIndexBuilder.cleanup's improveConnections): the batch's rows are written, then the back-link pairs (t, u), skipping
a pair when t's row (its new row if t is in the batch) already names u, sorted; pair i of t's segment lands at deg_before[t] + rank or
is dropped at row_cap; the rows past hard_max are re-pruned; after the last batch every row longer than M is re-pruned.
Compactor form (OnDiskGraphIndexCompactor's refine): every search reads the level as given, the rows replace the old ones at the end,
no back-links, beam 8 M.

Which nodes: builder form, at level 0 every member of level 1 and at each level L >= 1 every member of L, each with a non-empty row
there (in the graph as given); a flat graph is returned unchanged. Compactor form: level 0 only, the members of level 1, or every
node that is not a hole when the graph is flat.

Near ties: an F32Scores prune flags a row whose decision is a near tie (delete_model.pair_bound). In the compactor form no row
depends on another's prune (every search reads the given level), so a flagged prune leaves only its own row uncertain: the rows are
flagged one by one ("row_flags"). In the builder form every later batch searches the rows a flagged prune wrote, so a level whose model
made one has no single correct adjacency; it is reported as flagged (the level's count of flagged prunes)."""
import ctypes as C

import numpy as np

import graph_model as gm
import oracle_lib as o
from oracle_lib import fp, ip

BUILDER, COMPACTOR = 0, 1


def compactor_beam(M):
    """OnDiskGraphIndexCompactor's refine beam: 2 * max(M, max(2, 4 M))"""
    return 2 * max(M, max(2, 4 * M))


def union(row, results):
    """the row's valid entries in order, then the results that are not among them"""
    own = [int(x) for x in row if x >= 0]
    seen = set(own)
    return own + [int(x) for x in results if x >= 0 and int(x) not in seen]


class RefineModel(gm.BuildModel):
    def __init__(self, scores, M, beam, overflow, alpha, max_batch, rows, entry, compactor):
        super().__init__(scores, M, beam, overflow=overflow, alpha=alpha, max_batch=max_batch, window=0, rows=rows, entry=entry)
        self.compactor = compactor
        self.row_flags = {}  # node -> whether the prune that wrote its refined row was a near tie
        self.stats = {"candidates": 0, "max_candidates": 0, "backlinks_added": 0, "rows_repruned": 0}

    def search_excluding(self, u):
        g = o.make_graph(self.adj, self.entry)
        sf = self.scores.scorer(u)
        accept = np.ones(self.n, bool)
        accept[u] = False
        bits = gm.pack_bits(accept)
        nodes = np.full(self.beam, -1, np.int32)
        scores = np.zeros(self.beam, np.float32)
        cnt = self.L.jvo_graph_search_ex(C.byref(g), sf, None, self.beam, self.beam, 0.0, 0.0, bits.ctypes.data_as(C.POINTER(C.c_uint32)),
                                         ip(nodes), fp(scores), None)
        self.L.jvo_scorer_free(sf)
        return [int(x) for x in nodes[:cnt] if x >= 0]

    def candidates(self, u):
        return union(self.adj[u, :min(int(self.deg[u]), self.row_cap)], self.search_excluding(u))

    def apply_list(self, ids, rows, rdeg):
        """the batch's rows replace those of ids, then their back-links; returns the sorted list of rows that passed hard_max"""
        pos = {int(u): i for i, u in enumerate(ids)}
        for i, u in enumerate(ids):
            self.adj[u] = -1
            self.adj[u, :self.degree] = rows[i]
            self.deg[u] = rdeg[i]
        pairs = []
        for i, u in enumerate(ids):
            u = int(u)
            for t in rows[i]:
                t = int(t)
                if t < 0:
                    continue
                trow = rows[pos[t]] if t in pos else self.adj[t]
                if u in set(int(x) for x in trow):
                    continue
                pairs.append((t, u))
        pairs.sort()
        over, k = [], 0
        while k < len(pairs):
            t = pairs[k][0]
            e = k
            while e < len(pairs) and pairs[e][0] == t:
                e += 1
            d0 = int(self.deg[t])
            for r in range(e - k):
                if d0 + r < self.row_cap:
                    self.adj[t, d0 + r] = pairs[k + r][1]
                    self.stats["backlinks_added"] += 1
                else:
                    self.dropped += 1
            nd = min(self.row_cap, d0 + e - k)
            self.deg[t] = nd
            if nd > self.hard_max:
                over.append(t)
            k = e
        return over

    def refine(self, nodes):
        """refines the ascending rows `nodes`; returns the level's adjacency [n][M]"""
        nodes = [int(v) for v in nodes]
        kept = []
        for b0 in range(0, len(nodes), self.max_batch):
            batch = nodes[b0:b0 + self.max_batch]
            rows = np.full((len(batch), self.degree), -1, np.int32)
            rdeg = np.zeros(len(batch), np.int32)
            for i, u in enumerate(batch):
                c = self.candidates(u)
                self.stats["candidates"] += len(c)
                self.stats["max_candidates"] = max(self.stats["max_candidates"], len(c))
                sel, flag = self.prune(u, c)
                self.row_flags[u] = bool(flag)
                rows[i, :len(sel)] = sel
                rdeg[i] = len(sel)
            if self.compactor:
                kept.append((batch, rows, rdeg))
                continue
            over = self.apply_list(batch, rows, rdeg)
            self.stats["rows_repruned"] += len(over)
            self.apply_repruned(over, *self.reprune_rows(over)[:2])
        if self.compactor:
            for batch, rows, rdeg in kept:
                for i, u in enumerate(batch):
                    self.adj[u] = -1
                    self.adj[u, :self.degree] = rows[i]
                    self.deg[u] = rdeg[i]
        else:
            over = self.over_degree()
            self.stats["rows_repruned"] += len(over)
            self.apply_repruned(over, *self.reprune_rows(over)[:2])
        return self.compact()


def refine_graph(scores, levels, entry, holes, M, beam, overflow, alpha, max_batch, mode):
    """the refine of a graph given as levels [(ids, adj in node ids)] (level 0 first, its ids arange(n)), its entry and holes (bool [n]).
    Returns {"levels": [(ids, adj, flagged prunes)], "row_flags": per level {row: near tie of the prune that refined it}, "stats":
    jv_refine_stats' counters, "nodes_refined": per level}"""
    compactor = mode == COMPACTOR
    beam = compactor_beam(M) if compactor else beam
    n = levels[0][1].shape[0]
    out = [(ids, adj, 0) for ids, adj in levels]
    stats = {"levels": 0, "candidates": 0, "max_candidates": 0, "rows_changed": 0, "backlinks_added": 0, "backlinks_dropped": 0,
             "rows_repruned": 0}
    nodes_refined, row_flags = [], [{} for _ in levels]
    if entry < 0 or (not compactor and len(levels) == 1):
        return {"levels": out, "row_flags": row_flags, "stats": stats, "nodes_refined": nodes_refined}
    for lv in range(1 if compactor else len(levels)):
        ids, adj = levels[lv]
        nonempty = (adj >= 0).any(1)
        if lv == 0:
            if len(levels) > 1:
                nodes = [int(v) for v in levels[1][0] if compactor or nonempty[v]]
            else:
                nodes = [v for v in range(n) if not holes[v]]
            nodes.sort()
            sub, local, at = scores, adj, entry
        else:
            nodes = [r for r in range(len(ids)) if nonempty[r]]
            pos = np.full(n, -1, np.int64)
            pos[ids] = np.arange(len(ids))
            local = np.where(adj >= 0, pos[np.clip(adj, 0, None)], -1).astype(np.int32)
            sub, at = scores.subset(ids), int(pos[entry]) if pos[entry] >= 0 else 0
        nodes_refined.append(len(nodes))
        if not nodes:
            continue
        model = RefineModel(sub, M, beam, overflow, alpha, max_batch, local, at, compactor)
        new = model.refine(nodes)
        if lv > 0:
            new = np.where(new >= 0, ids[np.clip(new, 0, None)], -1).astype(np.int32)
        out[lv] = (ids, new, model.flagged)
        row_flags[lv] = model.row_flags
        for k in ("candidates", "backlinks_added", "rows_repruned"):
            stats[k] += model.stats[k]
        stats["max_candidates"] = max(stats["max_candidates"], model.stats["max_candidates"])
        stats["backlinks_dropped"] += model.dropped
        stats["rows_changed"] += int((new != adj).any(1).sum())
    stats["levels"] = len(nodes_refined)
    return {"levels": out, "row_flags": row_flags, "stats": stats, "nodes_refined": nodes_refined}
