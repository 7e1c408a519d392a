"""The device builder (jv_builder_*) driven step by step, the way parallel.sharded_build drives it on one GPU, against the host model
(graph_model.BuildModel), and the helpers the graph tests share. Needs a GPU."""
import ctypes as C

import numpy as np

import delete_model as dm
import graph_model as gm


def ptr(t):
    return C.c_void_p(t.data_ptr())


def levels(gi):
    return [gi.level(lv) for lv in range(gi.info()["levels"])]


def bits(mask):
    """bool [n] of marked (or deleted) nodes -> the uint32 words the jv_* calls take; None stays None"""
    from jvector_b200.api import pack_accept_bits
    return pack_accept_bits(mask).ctypes.data_as(C.POINTER(C.c_uint32)) if mask is not None else None


def assert_same_graph(a, b, what):
    ia, ib = a.info(), b.info()
    assert ia == ib, (what, ia, ib)
    for lv, ((ids_a, adj_a), (ids_b, adj_b)) in enumerate(zip(levels(a), levels(b))):
        assert np.array_equal(ids_a, ids_b) and np.array_equal(adj_a, adj_b), (what, "level", lv)


def builder(jv, metric, M, beam=60, hier=False, seed=3, **kw):
    return jv.GraphIndexBuilder(metric, M=M, beamWidth=beam, neighborOverflow=1.2, alpha=1.2, addHierarchy=hier, seed=seed, **kw)


def model_kw(params):
    """the BuildModel arguments of a jv_build_params"""
    return dict(M=params.degree, beam=params.beam_width, overflow=params.overflow, alpha=params.alpha, max_batch=params.max_batch,
                window=params.concurrent_window)


def _stream():
    import torch
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _compare(got, gdeg, want, wdeg, flags, what):
    """rows the model did not flag must be equal; returns (rows, flagged, differing)"""
    differ = (got != want).any(1) | (gdeg != wdeg)
    bad = np.flatnonzero(differ & ~flags)
    assert len(bad) == 0, (what, "rows differ", bad[:5].tolist(), got[bad[:1]].tolist(), want[bad[:1]].tolist())
    return len(flags), int(flags.sum()), int(differ.sum())


def drive(lib, b, model, cid, slices=2):
    """the created builder b driven to the end against `model` (in the builder's state), then freed: jv_builder_info and every batch
    equal the model's; every other batch is inserted in `slices` slices; each batch's inserted rows, overflow list and re-pruned rows
    equal the model's except rows it flags, and the mirror then adopts the device's rows (a flagged near tie cannot cascade); at the
    end the counters and the compacted adjacency. Returns (GraphIndex, tally {"insert", "reprune": [rows, flagged, differing]},
    batches)"""
    import torch

    import jvector_b200 as jv
    from jvector_b200 import _native as nat
    tally = {"insert": [0, 0, 0], "reprune": [0, 0, 0]}

    def add(kind, r):
        tally[kind] = [a + x for a, x in zip(tally[kind], r)]

    def reprune_round(L, lst, what):
        assert L == len(lst), (what, "rows to re-prune", L, len(lst))
        if L == 0:
            return
        rp = torch.empty((L, model.row_cap), dtype=torch.int32, device="cuda")
        rpd = torch.empty(L, dtype=torch.int32, device="cuda")
        nat.check(lib.jv_builder_reprune_slice(b, 0, L, ptr(rp), ptr(rpd)))
        got, gdeg = rp.cpu().numpy(), rpd.cpu().numpy()
        want, wdeg, flags = model.reprune_rows(lst)
        add("reprune", _compare(got, gdeg, want, wdeg, flags, what))
        model.apply_repruned(lst, got, gdeg)
        nat.check(lib.jv_builder_apply_repruned(b, L, ptr(rp), ptr(rpd)))

    first, count, L = C.c_int32(), C.c_int32(), C.c_int32()
    batches = 0
    try:
        deg_, cap_, mb_ = C.c_int(), C.c_int(), C.c_int()
        nat.check(lib.jv_builder_info(b, C.byref(deg_), C.byref(cap_), C.byref(mb_)))
        assert (deg_.value, cap_.value) == (model.degree, model.row_cap), (cid, deg_.value, cap_.value)
        rows_t = torch.empty((mb_.value, model.degree), dtype=torch.int32, device="cuda")
        rdeg_t = torch.empty(mb_.value, dtype=torch.int32, device="cuda")
        while True:
            nat.check(lib.jv_builder_next_batch(b, C.byref(first), C.byref(count)))
            f, c = first.value, count.value
            if c == 0:
                assert model.next_batch() is None
                break
            assert (f, c) == model.next_batch()
            # every other batch in slices: rows land at out_base + i, nodes are node_base + i
            cuts = [c * i // slices for i in range(slices + 1)] if batches % 2 else [0, c]
            for lo, hi in zip(cuts, cuts[1:]):
                nat.check(lib.jv_builder_insert_slice(b, f, c, lo, hi, ptr(rows_t), ptr(rdeg_t)))
            got, gdeg = rows_t[:c].cpu().numpy(), rdeg_t[:c].cpu().numpy()
            want, wdeg, flags = model.insert_rows(f, c)
            add("insert", _compare(got, gdeg, want, wdeg, flags, (cid, "batch", batches, f, c)))
            nat.check(lib.jv_builder_apply_new(b, f, c, ptr(rows_t), ptr(rdeg_t), C.byref(L)))
            reprune_round(L.value, model.apply_new(f, c, got, gdeg), (cid, "batch", batches))
            batches += 1
        nat.check(lib.jv_builder_collect_over_degree(b, C.byref(L)))
        reprune_round(L.value, model.over_degree(), (cid, "cleanup"))
        s = [C.c_int64() for _ in range(3)]
        nat.check(lib.jv_builder_stats(b, *[C.byref(x) for x in s]))
        h = C.c_void_p()
        nat.check(lib.jv_builder_finish(b, C.byref(h), None))
    finally:
        lib.jv_builder_free(b)
    gi = jv.GraphIndex(_handle=h)
    stats = tuple(x.value for x in s)
    assert stats == (batches, 0, model.dropped), (cid, stats, model.dropped)
    assert np.array_equal(gi.level(0)[1], model.compact()), (cid, "finished adjacency")
    return gi, tally, batches


def check_levels(gi, want_levels, want_entry, what):
    """the upper levels [(ids, adj, flagged prunes)] and the entry: a level the model built without a near tie has one correct
    adjacency. Returns (levels compared, levels skipped for a near tie)"""
    inf = gi.info()
    assert inf["entry_node"] == want_entry and inf["levels"] == 1 + len(want_levels), (what, inf, want_entry, len(want_levels))
    checked = 0
    for lv, (ids, want_adj, flagged) in enumerate(want_levels, 1):
        gids, gadj = gi.level(lv)
        assert np.array_equal(gids, ids), (what, "members of level", lv)
        if flagged == 0:
            assert np.array_equal(gadj, want_adj), (what, "level", lv)
            checked += 1
    return checked, len(want_levels) - checked


def drive_build(lib, ds, metric, params, make_scores, cid, suffix=""):
    """the build of ds through jv_builder_create<suffix>, driven against the model over make_scores() (called once the builder exists:
    a PQ builder makes the data set's pair table), then the upper levels and entry. Returns (GraphIndex, tally, batches, dropped
    back-links, (upper levels compared, skipped))"""
    from jvector_b200 import _native as nat
    b = C.c_void_p()
    nat.check(getattr(lib, "jv_builder_create" + suffix)(ds._h, metric, C.byref(params), _stream(), C.byref(b)))
    scores = make_scores()
    kw = model_kw(params)
    model = gm.BuildModel(scores, **kw)
    gi, tally, batches = drive(lib, b, model, cid)
    upper = (0, 0)
    if params.add_hierarchy:
        members, entry = gm.assign_levels(scores.n, params.degree, params.seed)
        upper = check_levels(gi, gm.upper_levels(scores, members, **kw), entry, cid)
    return gi, tally, batches, model.dropped, upper


def check_one_call_add(lib, g, ds, metric, params, marks, gi, batches, dropped, what, suffix="", metrics=None):
    """jv_graph_add_nodes<suffix> in one call gives the step-wise add's bytes, call after call (at each of `metrics`; default the add's
    own metric twice), with its batch and drop counters"""
    import jvector_b200 as jv
    from jvector_b200 import _native as nat
    ms = C.c_double()
    for m in metrics or (metric, metric):
        h = C.c_void_p()
        nat.check(getattr(lib, "jv_graph_add_nodes" + suffix)(g._h, ds._h, m, C.byref(params), bits(marks), C.byref(h), C.byref(ms)))
        one = jv.GraphIndex(_handle=h)
        assert_same_graph(gi, one, (what, "step-wise vs one call", m))
        one.close()
        sv, nb, nd = C.c_int64(), C.c_int64(), C.c_int64()
        lib.jv_graph_build_stats(C.byref(sv), C.byref(nb), C.byref(nd))
        assert (nb.value, nd.value) == (batches, dropped) and sv.value > 0 and ms.value > 0, (what, sv.value, nb.value, nd.value)


def drive_add(lib, g, ds, metric, params, marks, make_scores, cid, suffix="", metrics=None, slices=2):
    """the add of rows [n0, n) of ds to g through jv_builder_create_from_graph<suffix>, driven against the seeded model over
    make_scores() (called once the builder exists); then the upper levels and entry, the one-call add (check_one_call_add), and no
    new row naming a marked node. marks: bool [n0] or None. Returns (GraphIndex, tally, batches, dropped back-links, (upper levels
    compared, skipped))"""
    from jvector_b200 import _native as nat
    n0, entry0, levels0 = g.info()["n"], g.info()["entry_node"], levels(g)
    b = C.c_void_p()
    nat.check(getattr(lib, "jv_builder_create_from_graph" + suffix)(g._h, ds._h, metric, C.byref(params), bits(marks), _stream(), C.byref(b)))
    scores = make_scores()
    n, kw = scores.n, model_kw(params)
    accept = None if marks is None else np.concatenate([~marks, np.ones(n - n0, bool)])
    model = gm.BuildModel(scores, rows=levels0[0][1], entry=entry0, accept=accept, **kw)
    gi, tally, batches = drive(lib, b, model, cid, slices)
    upper = (0, 0)
    if len(levels0) > 1:
        upper = check_levels(gi, *gm.extend_levels(scores, levels0[1:], entry0, n0, params.seed, marks, **kw), cid)
    else:
        inf = gi.info()
        assert inf["levels"] == 1 and inf["entry_node"] == model.entry, (cid, inf, model.entry)
    check_one_call_add(lib, g, ds, metric, params, marks, gi, batches, model.dropped, cid, suffix, metrics)
    if marks is not None:
        marked = np.concatenate([marks, np.zeros(n - n0, bool)])
        for lv, (ids, ladj) in enumerate(levels(gi)):
            new_rows = ladj[ids >= n0]
            assert not marked[new_rows[new_rows >= 0]].any(), (cid, "a new row names a marked node on level", lv)
    return gi, tally, batches, model.dropped, upper


def step_build(ds, metric, params, suffix=""):
    """jv_builder_create<suffix> + jv_builder_* without a model: (GraphIndex, (batches, truncated, dropped))"""
    import torch

    import jvector_b200 as jv
    from jvector_b200 import _native as nat
    lib = nat.init()
    b = C.c_void_p()
    nat.check(getattr(lib, "jv_builder_create" + suffix)(ds._h, metric, C.byref(params), _stream(), C.byref(b)))
    try:
        deg_, cap_, mb_ = C.c_int(), C.c_int(), C.c_int()
        nat.check(lib.jv_builder_info(b, C.byref(deg_), C.byref(cap_), C.byref(mb_)))
        rows = torch.empty((mb_.value, deg_.value), dtype=torch.int32, device="cuda")
        rdeg = torch.empty(mb_.value, dtype=torch.int32, device="cuda")
        first, count, L = C.c_int32(), C.c_int32(), C.c_int32()

        def reprune(L):
            if L:
                rp = torch.empty((L, cap_.value), dtype=torch.int32, device="cuda")
                rpd = torch.empty(L, dtype=torch.int32, device="cuda")
                nat.check(lib.jv_builder_reprune_slice(b, 0, L, ptr(rp), ptr(rpd)))
                nat.check(lib.jv_builder_apply_repruned(b, L, ptr(rp), ptr(rpd)))

        while True:
            nat.check(lib.jv_builder_next_batch(b, C.byref(first), C.byref(count)))
            if count.value == 0:
                break
            nat.check(lib.jv_builder_insert_slice(b, first.value, count.value, 0, count.value, ptr(rows), ptr(rdeg)))
            nat.check(lib.jv_builder_apply_new(b, first.value, count.value, ptr(rows), ptr(rdeg), C.byref(L)))
            reprune(L.value)
        nat.check(lib.jv_builder_collect_over_degree(b, C.byref(L)))
        reprune(L.value)
        s = [C.c_int64() for _ in range(3)]
        nat.check(lib.jv_builder_stats(b, *[C.byref(x) for x in s]))
        g = C.c_void_p()
        nat.check(lib.jv_builder_finish(b, C.byref(g), None))
    finally:
        lib.jv_builder_free(b)
    return jv.GraphIndex(_handle=g), tuple(x.value for x in s)


def assert_removal_matches_model(gi, res, what):
    """a removal equals delete_model.remove_deleted's result row for row, with its counters; returns the repaired rows per code tier"""
    inf = gi.info()
    assert inf["entry_node"] == res["entry"] and inf["levels"] == res["levels"], (what, inf, res["entry"], res["levels"])
    want = [(np.arange(res["adj0"].shape[0], dtype=np.int32), res["adj0"])] + list(res["upper"])
    for L, ((dids, dadj), (wids, wadj)) in enumerate(zip(levels(gi), want)):
        assert np.array_equal(dids, wids), (what, "members of level", L)
        bad = np.flatnonzero((dadj != wadj).any(1))
        assert len(bad) == 0, (what, "level", L, "rows differ", wids[bad[:5]].tolist(), dadj[bad[:1]].tolist(), wadj[bad[:1]].tolist())
    cands = [len(r["cands"] - {v}) for lv in res["rows"] for v, r in lv.items()]
    st = gi.remove_stats
    assert st["repaired_rows"] == len(cands) and st["candidates"] == sum(cands) and st["max_candidates"] == max(cands, default=0), (what, st)
    assert st["random_fallbacks"] == sum(r["fallback"] for lv in res["rows"] for r in lv.values()), (what, st)
    assert st["live_nodes"] == (~res["dead"]).sum()
    return np.bincount([dm.repair_tier(c) for c in cands], minlength=len(dm.CODE_REPAIR_TIERS))
