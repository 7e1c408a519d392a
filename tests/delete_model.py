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
fp32. Pair similarities (the isDiverse test) carry the proven bound of pair_bound: a test is a near tie when score(c) * alpha lies
between the running maxima of (similarity - bound) and (similarity + bound). Without the device's key scores, two adjacent sorted
candidate scores equal within relative REL are near ties too. Only on flagged rows may the device (fp32 keys, 3xTF32 Gram products)
legitimately disagree. Given the device's own key scores (key_scores, the oracle's warp-order scorer) the candidate order is
certain, and only isDiverse tests are flagged."""
import numpy as np

EUCLIDEAN, DOT_PRODUCT, COSINE = 0, 1, 2
REL = 1e-5
U = 2.0 ** -24  # fp32 unit round-off
# 3xTF32 (prune_gram_tc_kernel): the dropped lo * lo product and the tf32 truncation of lo in the two cross products, each below
# 2^-20 |x_k y_k| (|lo| < 2^-10 |x|): 3 * 2^-20 relative to |x| |y| over the whole sum
TF32_SPLIT = 3 * 2.0 ** -20
_M64 = (1 << 64) - 1


def dot_gamma(stride):
    """relative error of any fp32 dot product of depth below stride + 8, whatever the summation order (DESIGN §4.1), plus the
    3xTF32 split of the tensor-core Gram product"""
    return (stride + 8) * 2.0 ** -23 + TF32_SPLIT


def pair_bound(metric, X, xv, stride):
    """[nc][nc] bound on |device pair similarity - exact pair similarity| for the candidate rows X (float64) of the node whose
    row is xv, for every prune tier (fp32 Gram product on the CUDA or the tensor cores, or the direct fp32 sum of prune_kernel).
    DOT / COSINE: the dot product's error gamma |x_i| |x_j| through the score map. L2: gamma (|x_i - x_v| + |x_j - x_v|)^2 on the
    squared distance, which bounds the direct sum (|x_i - x_j| <= |x_i - x_v| + |x_j - x_v|) and the Gram form over rows translated
    by x_v (build.cu gram_row); it does not depend on how far the rows sit from the origin."""
    g = dot_gamma(stride) + 4 * U  # + the rounding of the translation and of the final adds
    if metric == EUCLIDEAN:
        Y = X - xv
        r = np.sqrt((Y * Y).sum(1))
        dd = g * (r[:, None] + r[None, :]) ** 2
        if np.array_equal(Y, np.round(Y)) and np.abs(Y).max(initial=0) < 2048:
            # integer rows (SIFT): every product and partial sum is an integer below 2^24 while (r_i + r_j)^2 is, so the pair's
            # squared distance is exact in fp32 on every tier (integers below 2^11 have no 3xTF32 lo part)
            dd = np.where((r[:, None] + r[None, :]) ** 2 < 2.0 ** 24, 0.0, dd)
        d = _sqdist(Y)
        return dd / ((1.0 + d) * (1.0 + np.maximum(0.0, d - dd))) + 4 * U / (1.0 + d)
    nrm = np.sqrt((X * X).sum(1))
    if metric == DOT_PRODUCT:
        return g * nrm[:, None] * nrm[None, :] / 2.0 + 2 * U * np.abs(1.0 + X @ X.T) + 4 * U
    # cosine: g from the dot product, g / 2 from each squared norm under the square root, then the divide
    return np.full((len(X), len(X)), (2 * g + 4 * U) / 2.0 + 4 * U)


def _sqdist(Y):
    """squared distances of the rows of Y (float64; translated by the pruned node's row, so the Gram form loses nothing)"""
    n2 = (Y * Y).sum(1)
    return np.maximum(0.0, n2[:, None] + n2[None, :] - 2.0 * (Y @ Y.T))


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


def _pairs(metric, Y, xv):
    if metric == EUCLIDEAN:
        return 1.0 / (1.0 + _sqdist(Y - xv))
    G = Y @ Y.T
    if metric == DOT_PRODUCT:
        return (1.0 + G) / 2.0
    d = np.diag(G)
    return (1.0 + G / np.sqrt(d[:, None] * d[None, :])) / 2.0


def retain_diverse(metric, data, v, cands, degree, alpha, key_scores=None):
    """retainDiverse with diverseBefore = 0 over the distinct `cands` of node v: (selected ids in score order, near-tie flag).
    key_scores(v, ids) -> float32: the candidates' scores against v with the device's exact bits (the oracle's warp-order
    scorer); then their order is certain and only the isDiverse tests can be near ties. Without it, exact float64 scores."""
    c = np.array(sorted(set(int(x) for x in cands) - {int(v)}), dtype=np.int64)
    if len(c) == 0:
        return [], False
    X = data[c].astype(np.float64)
    xv = data[v].astype(np.float64)
    s = _scores(metric, xv, X) if key_scores is None else np.asarray(key_scores(v, c), np.float32)
    order = np.lexsort((c, -s))  # score descending, then the lower id first
    c, s, X = c[order], s[order], X[order]
    flag = key_scores is None and any(_near(s[i], s[i + 1]) for i in range(len(s) - 1))
    P = _pairs(metric, X, xv)
    B = pair_bound(metric, X, xv, (data.shape[1] + 3) & ~3)
    maxsim = np.full(len(c), -np.inf)
    lo, hi = maxsim.copy(), maxsim.copy()  # running maxima of P - B and P + B: where the device's fp32 maximum can lie
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
            if lo[i] <= thr < hi[i]:
                flag = True
            if not maxsim[i] > thr:
                taken[i] = True
                sel.append(i)
                maxsim = np.maximum(maxsim, P[:, i])
                lo = np.maximum(lo, P[:, i] - B[:, i])
                hi = np.maximum(hi, P[:, i] + B[:, i])
        a = np.float32(a + np.float32(0.2))
    return [int(c[i]) for i in sorted(sel)], flag


# the capacities of the removal's prune over PQ or BQ codes (build.cu CODE_REPAIR_TIER_MAX): a row runs at the smallest that holds
# its candidates
CODE_REPAIR_TIERS = (64, 128, 256, 1024, 2048, 8192)


def repair_tier(ncand):
    return next(t for t, cap in enumerate(CODE_REPAIR_TIERS) if ncand <= cap or cap == CODE_REPAIR_TIERS[-1])


def remove_deleted(data, metric, adj0, entry, upper, deleted, alpha=1.2, seed=0, holes=None, key_scores=None, prune=None):
    """adj0 [n][degree]; upper: list of (ids, adj [count][degree], global ids) for levels 1..; deleted, holes: bool [n].
    key_scores: see retain_diverse. prune(v, cands, degree, alpha) -> (selected ids, near-tie flag): the row prune, by default
    retain_diverse over data (graph_model's score providers give the PQ and BQ ones).
    Returns {"adj0", "upper", "entry", "levels", "rows"}: rows[level][node] = {"flag", "fallback", "cands"} for every repaired row."""
    data = np.asarray(data, dtype=np.float32)
    if prune is None:
        def prune(v, cands, degree, alpha):
            return retain_diverse(metric, data, v, cands, degree, alpha, key_scores)
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
            sel, flag = prune(v, cands, degree, alpha)
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
