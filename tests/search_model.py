"""Host MODEL of graph_search_kernel's data structures (jvector_b200/csrc/search.cu), in plain Python — TEST INFRASTRUCTURE.

The kernel does not keep the reference's two heaps + evicted list; it keeps ONE sorted list of seen nodes (flags: expanded,
accepted) with a bounded length `list_cap`, plus a shadow copy of the reference's bounded result heap. The claim that this is
EXACTLY GraphSearcher.search — ties, upper levels, acceptOrds / threshold / rerankFloor, NodeQueue.rerank's array order —
is checked here on the CPU against the oracle's literal restatement (oracle/jv_oracle.c jvo_graph_search_ex), so that the
equivalence argument is pinned before any GPU time is spent. Each step below names the kernel code it mirrors."""
import numpy as np

F_EXPANDED, F_ACCEPTED = 1, 2
KEY_MIN = -(1 << 63)


class ListOverflow(Exception):
    """overflow code 2 of the kernel: the tie tail (or the filtered-out candidates) did not fit list_cap"""


def f2sortable(score):
    b = int(np.float32(score).view(np.int32))
    return b ^ ((b >> 31) & 0x7fffffff)


def topk_key(score, node):
    return (f2sortable(score) << 32) | ((~int(node)) & 0xffffffff)


def key_node(key):
    return (~key) & 0xffffffff


def key_score(key):
    s = key >> 32
    b = s ^ ((s >> 31) & 0x7fffffff)
    return float(np.int32(b).view(np.float32))


def heap_up(h, pos):  # AbstractLongHeap.upHeap; h is 1-based (h[0] unused)
    i, v = pos, h[pos]
    j = i >> 1
    while j > 0 and v < h[j]:
        h[i] = h[j]
        i, j = j, j >> 1
    h[i] = v


def heap_down(h, size, pos):  # AbstractLongHeap.downHeap
    i, v = pos, h[pos]
    j, k = i << 1, (i << 1) + 1
    if k <= size and h[k] < h[j]:
        j = k
    while j <= size and h[j] < v:
        h[i] = h[j]
        i = j
        j, k = i << 1, (i << 1) + 1
        if k <= size and h[k] < h[j]:
            j = k
    h[i] = v


def search(graph_levels, entry_node, score_fn, topK, rerankK, list_cap, rerank_fn=None, threshold=0.0, rerank_floor=0.0, accept=None):
    """graph_levels[l] = dict node -> list of neighbours (level 0 first); returns (nodes, scores, visited, reranked)."""
    L, LC = rerankK, list_cap
    assert LC >= L
    filtered = accept is not None or threshold > 0

    def accepted(node, sc):
        return (accept is None or bool(accept[node])) and sc >= np.float32(threshold)

    seen = {entry_node}
    es = score_fn(entry_node)
    lst = [[topk_key(es, entry_node), F_ACCEPTED if accepted(entry_node, es) else 0]]  # sorted by key, descending
    visited = 0
    heap = [0]
    for lvl in range(len(graph_levels) - 1, -1, -1):
        K = 1 if lvl > 0 else L
        for e in lst:
            e[1] &= F_ACCEPTED
        heap = [0]
        while True:
            p = next((i for i, e in enumerate(lst) if not (e[1] & F_EXPANDED)), None)
            if p is None:
                break
            ckey = lst[p][0]
            hs = len(heap) - 1
            csc = np.float32(key_score(ckey))
            wsc = np.float32(key_score(heap[1])) if hs > 0 else np.float32(0)
            if hs >= K and csc < wsc:
                break
            node = key_node(ckey)
            action = 0
            # searchOneLayer's score >= threshold: F_ACCEPTED at level 0, threshold 0 with Bits.ALL on upper levels
            if (csc >= 0) if lvl > 0 else (lst[p][1] & F_ACCEPTED):
                action = 1 if hs < K else (2 if csc > wsc else 3)
            dead = p if (lvl > 0 and action in (0, 3)) else -1
            lst[p][1] |= F_EXPANDED
            if action == 1:
                heap.append(ckey)
                heap_up(heap, hs + 1)
            elif action == 2:
                heap[1] = ckey
                heap_down(heap, hs, 1)
            cands = []
            for f in graph_levels[lvl].get(node, []):
                if f < 0:
                    break
                if f in seen:
                    continue
                seen.add(f)
                sc = score_fn(f)
                cands.append([topk_key(sc, f), F_ACCEPTED if accepted(f, sc) else 0])
                visited += 1
            # merge: drop `dead`, keep the best LC, remember the best score that fell off
            merged = [e for i, e in enumerate(lst) if i != dead] + cands
            merged.sort(key=lambda e: -e[0])
            dropped = merged[LC:]
            merged = merged[:LC]
            drop = [f2sortable(key_score(e[0])) for e in dropped if (not (e[1] & F_EXPANDED)) or lvl > 0]
            if drop:
                dm = max(drop)
                if not filtered and key_score(merged[L - 1][0]) >= 0:
                    ok = f2sortable(key_score(merged[L - 1][0])) > dm
                else:
                    ok = sum(1 for e in merged if (e[1] & F_ACCEPTED) and f2sortable(key_score(e[0])) > dm) >= L
                if not ok:
                    raise ListOverflow()
            lst = merged
    hs = len(heap) - 1
    if rerank_fn is None:
        keys = sorted(heap[1:], reverse=True)[:topK]
        return [key_node(k) for k in keys], [key_score(k) for k in keys], visited, 0
    take = [np.float32(key_score(heap[1 + i])) >= np.float32(rerank_floor) for i in range(hs)]
    if not any(take) and hs > 0:
        bi, bs = 0, np.float32(key_score(heap[1]))
        for i in range(1, hs):
            s = np.float32(key_score(heap[1 + i]))
            if s > bs:
                bs, bi = s, i
        take[bi] = True
    exact = [topk_key(rerank_fn(key_node(heap[1 + i])), key_node(heap[1 + i])) if take[i] else KEY_MIN for i in range(hs)]
    nrr = sum(take)
    srt = sorted(exact, reverse=True)
    if not (nrr > topK and key_score(srt[topK - 1]) == key_score(srt[topK])):
        keys = srt[:min(nrr, topK)]
    else:
        rh = [0]
        for v in exact:
            if v == KEY_MIN:
                continue
            if len(rh) - 1 < topK:
                rh.append(v)
                heap_up(rh, len(rh) - 1)
            elif np.float32(key_score(v)) > np.float32(key_score(rh[1])):
                rh[1] = v
                heap_down(rh, len(rh) - 1, 1)
        keys = sorted(rh[1:], reverse=True)
    return [key_node(k) for k in keys], [key_score(k) for k in keys], visited, nrr


# ------------------------------------------------------------------------------------------------------------------------
# The visited set of the walk in shared memory (search.cu visited_insert_smem + the sizing rule of plan_search): 16-bit slots,
# region = high bits of a bijective hash of the id, tag = its low 15 bits, probes never leave their region.
# ------------------------------------------------------------------------------------------------------------------------
VIS_MUL = 0x9E3779B1


def visited_smem_plan(n, visited_cap, slots_env=None):
    """(slots_log, region_log, id_mask) as plan_search chooses them, or None when the walk keeps the global table"""
    bits = 15
    while (1 << bits) < n:
        bits += 1
    slots = slots_env if slots_env else visited_cap // 2
    slog = 0
    while (1 << slog) < slots:
        slog += 1
    while not slots_env and slog - (bits - 15) < 7 and slog < 14:
        slog += 1
    rlog = slog - (bits - 15)
    if slog < 10 or slog > 14 or rlog < 5:
        return None
    return slog, rlog, (1 << bits) - 1


class VisitedSmem:
    def __init__(self, slog, rlog, idmask):
        self.t = np.zeros(1 << slog, np.uint16)
        self.rlog, self.idmask = rlog, idmask
        self.failed = False

    def insert(self, v):
        """True = new (visited.add() returned true), False = seen before (or the region is full: self.failed)"""
        x = (int(v) * VIS_MUL) & 0xffffffff & self.idmask
        tag = x & 0x7fff
        val = tag | 0x8000
        rmask = (1 << self.rlog) - 1
        base = (x >> 15) << self.rlog
        h = ((tag * VIS_MUL) & 0xffffffff) >> (32 - self.rlog)
        for _ in range(rmask + 1):
            old = int(self.t[base + h])
            if old == 0:
                self.t[base + h] = val
                return True
            if old == val:
                return False
            h = (h + 1) & rmask
        self.failed = True
        return False


def pq_group_sum8(parts):
    """group_sum<8> of common.cuh on one candidate's 8 lane sums: xor butterfly 4, 2, 1 in float32; returns lane 0's value"""
    v = [np.float32(p) for p in parts]
    for o in (4, 2, 1):
        v = [np.float32(v[i] + v[i ^ o]) for i in range(8)]
    return v


def pq_fold8(parts):
    """pq_fold8 of scorers.cuh: the same tree written out for one thread"""
    p = [np.float32(x) for x in parts]
    f = np.float32
    return f(f(f(p[0] + p[4]) + f(p[2] + p[6])) + f(f(p[1] + p[5]) + f(p[3] + p[7])))
