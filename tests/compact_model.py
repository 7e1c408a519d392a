"""OnDiskGraphIndexCompactor's merge restated on the host, scalar and single-threaded, as the checker of jv_graph_compact.

Follows graph/disk/OnDiskGraphIndexCompactor.java for fp32 sources: searchTopK = max(2, ceil(M / S) * 4) (:877-890); for every
level L, every source s and every live member v of s at L (:978-1055) the candidates are v's live neighbours at L in s (:1207-1223)
and, from every other source t that has a level L, the searchTopK best live members of t at L: at L = 0 a search of t's graph
filtered by t's live nodes (:1241-1257), above it a greedy descent from t's entry down to L + 1 and a beam of searchTopK on L
(:1258-1293). Here that search is the oracle's (jvo_graph_search_ex with the warp-order scorer, which the device search equals id
for id) over t's sub-hierarchy from L up, the graph jv_graph_compact searches. retainDiverse at alpha (:1719-1760, the builder's
rule) is delete_model.retain_diverse.

Deliberate differences from the reference, shared with the device: when t has at most searchTopK live members at L they are all
candidates and no search runs (what an exhaustive search returns); equal scores put the lower new id first; when no source's
entry qualifies, the entry is the lowest new id of the top level; the merged graph has no holes.

A source is a dict: data [n][dim] float32, adj0 [n][degree], upper [(ids, adj)] for levels 1.. (adj in node ids), entry, live
(bool [n]: holes are not live) and map (int [n], new ids of the live nodes)."""
import ctypes as C

import numpy as np

import delete_model as dm
import oracle_lib as o
from oracle_lib import fp, ip


def search_top_k(degree, nsources):
    return max(2, -(-degree // nsources) * 4)


def members(src, level):
    """(node ids of the level in its order, adjacency rows)"""
    if level == 0:
        return np.arange(src["adj0"].shape[0], dtype=np.int32), src["adj0"]
    ids, adj = src["upper"][level - 1]
    return np.asarray(ids, np.int32), np.asarray(adj, np.int32)


def levels_of(src):
    return 1 + len(src["upper"])


def sub_search(oracle, metric, src, level, queries, K):
    """the K best live members of src's level `level` for every query: the search of src's hierarchy from that level up (node ids)"""
    ids, adj = members(src, level)
    pos = np.full(src["adj0"].shape[0], -1, np.int64)
    pos[ids] = np.arange(len(ids))

    def remap(a):
        a = np.asarray(a, np.int64)
        return np.ascontiguousarray(np.where(a >= 0, pos[np.clip(a, 0, None)], -1), np.int32)

    upper = [(remap(i), remap(a)) for i, a in src["upper"][level:]]
    g = o.make_graph(remap(adj), int(pos[src["entry"]]), upper or None)
    rows = np.ascontiguousarray(src["data"][ids], np.float32)
    accept = _bits(src["live"][ids])
    out = np.full((len(queries), K), -1, np.int32)
    for i, q in enumerate(queries):
        sf = oracle.jvo_scorer_f32(metric, fp(rows), len(ids), rows.shape[1], fp(np.ascontiguousarray(q, np.float32)))
        oracle.jvo_scorer_set_order(sf, 1)
        nodes = np.full(K, -1, np.int32)
        scores = np.zeros(K, np.float32)
        oracle.jvo_graph_search_ex(C.byref(g), sf, None, K, K, 0.0, 0.0, accept.ctypes.data_as(C.POINTER(C.c_uint32)), ip(nodes), fp(scores), None)
        oracle.jvo_scorer_free(sf)
        out[i] = np.where(nodes >= 0, ids[np.clip(nodes, 0, None)], -1)
    return out


def _bits(mask):
    m = np.asarray(mask, bool)
    pad = (-len(m)) % 32
    m = np.concatenate([m, np.zeros(pad, bool)])
    return np.ascontiguousarray(np.packbits(m, bitorder="little").view(np.uint32))


def warp_keys(oracle, metric, data):
    """the candidates' scores with the device's bits (warp-order oracle scorer): the sort order is then certain"""
    dim = data.shape[1]
    return lambda v, ids: np.array([oracle.jvo_compare_f32_warp(metric, fp(data[v]), fp(data[i]), dim) for i in ids], np.float32)


def compact(oracle, metric, sources, alpha=1.2):
    """returns {"rows", "levels": [(ids, adj)] (level 0 ids = arange), "entry", "flags": per level {new id: near tie}, "cands": per
    level {new id: candidate set}, "stats": searches / exhaustive / candidates / max_candidates / search_top_k / nodes / levels}"""
    S = len(sources)
    degree = sources[0]["adj0"].shape[1]
    K = search_top_k(degree, S)
    total = int(sum(s["live"].sum() for s in sources))
    dim = sources[0]["data"].shape[1]
    rows = np.zeros((total, dim), np.float32)
    for s in sources:
        live = np.flatnonzero(s["live"])
        rows[s["map"][live]] = s["data"][live]
    keys = warp_keys(oracle, metric, rows)
    stats = {"searches": 0, "exhaustive": 0, "candidates": 0, "max_candidates": 0, "search_top_k": K, "nodes": total}
    out_levels, flags, cands_out = [], [], []
    for L in range(max(levels_of(s) for s in sources)):
        live_at = []
        for s in sources:
            if L < levels_of(s):
                ids, _ = members(s, L)
                live_at.append(ids[s["live"][ids]])
            else:
                live_at.append(np.zeros(0, np.int32))
        if sum(len(x) for x in live_at) == 0:
            break
        # per target: {(source, node): candidate new ids}
        found = [dict() for _ in range(S)]
        for t, st in enumerate(sources):
            if L >= levels_of(st):
                continue
            queries = [(s, int(v)) for s in range(S) if s != t for v in live_at[s]]
            if not queries:
                continue
            if len(live_at[t]) <= K:
                stats["exhaustive"] += len(queries)
                every = st["map"][live_at[t]].tolist()
                for q in queries:
                    found[t][q] = every
                continue
            stats["searches"] += len(queries)
            res = sub_search(oracle, metric, st, L, [sources[s]["data"][v] for s, v in queries], K)
            for q, r in zip(queries, res):
                found[t][q] = [int(st["map"][x]) for x in r if x >= 0]
        level_rows, fl, cl = {}, {}, {}
        for s, src in enumerate(sources):
            if not len(live_at[s]):
                continue
            ids, adj = members(src, L)
            row_of = {int(v): r for r, v in enumerate(ids)}
            for v in live_at[s]:
                nv = int(src["map"][v])
                c = [int(src["map"][j]) for j in adj[row_of[int(v)]] if j >= 0 and src["live"][j]]
                for t in range(S):
                    if t != s and (s, int(v)) in found[t]:
                        c += found[t][(s, int(v))]
                assert len(set(c)) == len(c)
                stats["candidates"] += len(c)
                stats["max_candidates"] = max(stats["max_candidates"], len(c))
                sel, flag = dm.retain_diverse(metric, rows, nv, c, degree, alpha, keys)
                level_rows[nv] = sel + [-1] * (degree - len(sel))
                fl[nv], cl[nv] = flag, set(c)
        nids = np.array(sorted(level_rows), np.int32)
        out_levels.append((nids, np.array([level_rows[int(v)] for v in nids], np.int32).reshape(len(nids), degree)))
        flags.append(fl)
        cands_out.append(cl)
    top = len(out_levels) - 1
    entry = -1
    for s in sources:
        if levels_of(s) - 1 == top and s["entry"] >= 0 and s["live"][s["entry"]]:
            entry = int(s["map"][s["entry"]])
            break
    if entry < 0:
        entry = int(out_levels[top][0].min())
    stats["levels"] = len(out_levels)
    return {"rows": rows, "levels": out_levels, "entry": entry, "flags": flags, "cands": cands_out, "stats": stats}
