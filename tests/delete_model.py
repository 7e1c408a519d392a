"""removeDeletedNodes restated on the host, scalar and single-threaded, as the checker of jv_graph_remove_deleted.

Follows GraphIndexBuilder.removeDeletedNodes (base:graph/GraphIndexBuilder.java:689-799): per level, every live row that names a
deleted node gathers the live ids (other than itself) of its deleted neighbours' rows (:705-721); when there are none it tries
2 * degree random live members of the level (:743-759); ConcurrentNeighborMap.replaceDeletedNeighbors (:225-239) merges them with
the row's live neighbours and VamanaDiversityProvider.retainDiverse (:45-96) picks the new row. The entry node, if deleted, becomes
the lowest live id of the highest level with a live member (:769-786).

Deliberate differences from the reference, shared with the device: ties in score put the lower id first (the project's top-k key;
the reference uses hash-set order), the random fallback draws from the level's live members with the counter-based generator
repair_random (the reference uses ThreadLocalRandom over all ids), and the new entry is the lowest live id rather than the first in
the level's iteration order.

Scores are exact (float64 over the fp32 rows). A row is flagged as a near tie when one of its decisions is too close to call in
fp32: two adjacent sorted candidate scores, or a running maximum similarity and score(c) * alpha in the isDiverse test, equal
within relative REL. Only on flagged rows may the device (fp32 keys, 3xTF32 Gram products) legitimately disagree. Given the
device's own key scores (key_scores, the oracle's warp-order scorer) the candidate order is certain, and only isDiverse tests are
flagged: at 10 % deleted and M = 16 that leaves about 0.5 % of the repaired rows flagged, at 40 % and M = 32 about 0.7 %."""
import numpy as np

EUCLIDEAN, DOT_PRODUCT, COSINE = 0, 1, 2
REL = 1e-5
_M64 = (1 << 64) - 1


def _mix(x):
    x = (x + 0x9E3779B97F4A7C15) & _M64
    x = ((x ^ (x >> 30)) * 0xBF58476D1CE4E5B9) & _M64
    x = ((x ^ (x >> 27)) * 0x94D049BB133111EB) & _M64
    return x ^ (x >> 31)


def repair_random(seed, level, node, attempt):
    """the fallback's generator: a pure function of (seed, level, node, attempt) (repair_random in build.cu)"""
    return _mix(_mix(_mix((int(seed) ^ int(level)) & _M64) ^ int(node)) ^ int(attempt))


def _near(a, b):
    return abs(a - b) <= REL * max(abs(a), abs(b))


def _scores(metric, x, Y):
    if metric == EUCLIDEAN:
        return 1.0 / (1.0 + ((Y - x) ** 2).sum(1))
    if metric == DOT_PRODUCT:
        return (1.0 + Y @ x) / 2.0
    return (1.0 + (Y @ x) / np.sqrt((Y * Y).sum(1) * (x @ x))) / 2.0


def _pairs(metric, Y):
    G = Y @ Y.T
    if metric == EUCLIDEAN:
        d = np.diag(G)
        return 1.0 / (1.0 + np.maximum(0.0, d[:, None] + d[None, :] - 2.0 * G))
    if metric == DOT_PRODUCT:
        return (1.0 + G) / 2.0
    d = np.diag(G)
    return (1.0 + G / np.sqrt(d[:, None] * d[None, :])) / 2.0


def retain_diverse(metric, data, v, cands, degree, alpha, key_scores=None):
    """retainDiverse with diverseBefore = 0 over the distinct `cands` of node v: (selected ids in score order, near-tie flag).
    key_scores(v, ids) -> float32: the candidates' scores against v with the device's exact bits (the oracle's warp-order
    scorer); then their order is certain and only the isDiverse tests can be near ties. Without it, exact float64 scores."""
    c = np.array(sorted(set(int(x) for x in cands)), dtype=np.int64)
    if len(c) == 0:
        return [], False
    X = data[c].astype(np.float64)
    s = _scores(metric, data[v].astype(np.float64), X) if key_scores is None else np.asarray(key_scores(v, c), np.float32)
    order = np.lexsort((c, -s))  # score descending, then the lower id first
    c, s, X = c[order], s[order], X[order]
    flag = key_scores is None and any(_near(s[i], s[i + 1]) for i in range(len(s) - 1))
    P = _pairs(metric, X)
    maxsim = np.full(len(c), -np.inf)
    taken = np.zeros(len(c), bool)
    sel = []
    a = np.float32(1.0)
    lim = np.float32(np.float32(alpha) + np.float32(1e-6))
    while a <= lim and len(sel) < degree:
        for i in range(len(c)):
            if len(sel) >= degree:
                break
            if taken[i]:
                continue
            thr = float(np.float32(s[i]) * a) if key_scores is not None else s[i] * float(a)  # fp32 product, as __fmul_rn
            if np.isfinite(maxsim[i]) and _near(maxsim[i], thr):
                flag = True
            if not maxsim[i] > thr:
                taken[i] = True
                sel.append(i)
                maxsim = np.maximum(maxsim, P[:, i])
        a = np.float32(a + np.float32(0.2))
    return [int(c[i]) for i in sorted(sel)], flag


def remove_deleted(data, metric, adj0, entry, upper, deleted, alpha=1.2, seed=0, holes=None, key_scores=None):
    """adj0 [n][degree]; upper: list of (ids, adj [count][degree], global ids) for levels 1..; deleted, holes: bool [n].
    key_scores: see retain_diverse.
    Returns {"adj0", "upper", "entry", "levels", "rows"}: rows[level][node] = {"flag", "fallback", "cands"} for every repaired row."""
    data = np.asarray(data, dtype=np.float32)
    n, degree = adj0.shape
    dead = np.asarray(deleted, bool).copy()
    if holes is not None:
        dead |= np.asarray(holes, bool)
    levels = [(np.arange(n, dtype=np.int32), adj0)] + [(np.asarray(i, np.int32), np.asarray(a, np.int32)) for i, a in (upper or [])]
    out_upper, rows_info = [], []
    new0 = None
    for L, (ids, adj) in enumerate(levels):
        rowmap = np.full(n, -1, np.int64)
        rowmap[ids] = np.arange(len(ids))
        members = np.sort(ids[~dead[ids]])
        new = adj.copy()
        info = {}
        nbdead = np.where(adj >= 0, dead[np.clip(adj, 0, None)], False)
        for r in np.flatnonzero(nbdead.any(1) & ~dead[ids]):
            v = int(ids[r])
            row = adj[r]
            live = [int(j) for j in row if j >= 0 and not dead[j]]
            two = set()
            for j in row[nbdead[r]]:
                rj = rowmap[j]
                if rj < 0:
                    continue
                for k in adj[rj]:
                    if k >= 0 and k != v and not dead[k]:
                        two.add(int(k))
            fallback = not two
            if fallback:
                picks = []
                for at in range(2 * degree):
                    if len(picks) >= degree or len(members) == 0:
                        break
                    k = int(members[repair_random(seed, L, v, at) % len(members)])
                    if k != v and k not in picks:
                        picks.append(k)
                two = set(picks)
            cands = set(live) | two
            sel, flag = retain_diverse(metric, data, v, cands, degree, alpha, key_scores)
            new[r] = sel + [-1] * (degree - len(sel))
            info[v] = {"flag": flag, "fallback": fallback, "cands": cands}
        rows_info.append(info)
        if L == 0:
            new[dead] = -1
            new0 = new
        else:
            keep = ~dead[ids]
            out_upper.append((ids[keep].copy(), new[keep].copy()))
    e = int(entry)
    if e < 0 or dead[e]:
        e = -1
        while out_upper and len(out_upper[-1][0]) == 0:
            out_upper.pop()
        if out_upper:
            e = int(out_upper[-1][0].min())
        elif (~dead).any():
            e = int(np.flatnonzero(~dead)[0])
    return {"adj0": new0, "upper": out_upper, "entry": e, "levels": 1 + len(out_upper), "rows": rows_info, "dead": dead}
