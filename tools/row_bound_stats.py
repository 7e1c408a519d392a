#!/usr/bin/env python
"""How many bytes a row sketch would save the c2 walk: builds the c2 world the way bench.py does (1M x 768 latent rows, 10 000
queries, DOT_PRODUCT, topK 10, rerankK 100), runs one search on a counter build of the library (-DJV_ROW_BOUND_STATS, built here
with tools/build_variant.sh) and reports

    f = share of the level-0 rows the walk scores that JV_EMIT drops against a full candidate list,
    b = share of those drops that the sketch's upper bound (tests/row_bound_model.py) still catches,

for the fp16 sketch and for an int8 sketch with one scale per row; b is replayed on the host over a sample of the drops
({query, row, key of the list's last entry}). Predicted bytes per visited row = sketch + 8 + (1 - f b) 4 d, against 4 d + 8.

For the two-tier int8 sketch (tests/row_bound_coarse.py) it also reports b1, the share of the drops the coarse half's bound catches,
and b12, the share caught by the coarse or the int8 bound, and predicts (ss = sketch bytes per row)

    (ss / 2 + 16) + 8 + (1 - f b1) ss / 2 + (1 - f b12) 4 d    against the one-tier ss + 8 + 8 + (1 - f b) 4 d.

For the low-rank edge bound (tests/row_bound_lowrank.py, a basis fitted on --basis-rows sampled rows) at each k of --ranks it reports
b1, the share of the drops that bound catches before the sketch is read, and predicts

    rec + (1 - f b1) (ss + 16) + (1 - f b) 4 d,   rec = degree (k + 16) / (new rows per hop),

where rec counts the whole edge record of every expanded node (its k + 16 B slots stored with the adjacency row).

For the routing of the edge tier (a row the edge bound does not settle goes straight to its full row when the bound's point estimate,
tests/row_bound_direct.py point_estimate, scores more than delta above the list's last entry) it replays a 1-in-64 sample of every
row scored against a full list ({query, row, last key, exact key}) at each delta of --deltas, and reports the share of the list's
entrants routed direct, the share of the scored rows that are drops routed direct (each reads 4 d instead of ss + 16 B), and the
predicted bytes per scored row, rec + (ss + 16 for a row that reads its sketch) + (4 d for a row that reads its full row), against
the same replay with no row routed direct.

    python tools/row_bound_stats.py [--out row_bound_stats.json]"""
import argparse
import json
import os
import subprocess
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
VARIANT = os.path.join(ROOT, "jvector_b200", "lib_rbs", "libjvector_b200.so")

ap = argparse.ArgumentParser()
ap.add_argument("--n", type=int, default=1_000_000)
ap.add_argument("--nq", type=int, default=10_000)
ap.add_argument("--max-samples", type=int, default=100_000)
ap.add_argument("--ranks", default="16,32,64")
ap.add_argument("--basis-rows", type=int, default=4096)
ap.add_argument("--deltas", default="0,0.0005,0.001,0.002,0.003,0.004,0.005,0.0075,0.01,0.015,0.02")
ap.add_argument("--out", default="")
a = ap.parse_args()

if not os.path.exists(VARIANT):
    subprocess.run([os.path.join(ROOT, "tools", "build_variant.sh"), "rbs", "-DJV_ROW_BOUND_STATS"], check=True, stdout=subprocess.DEVNULL)
os.environ["JV_B200_SO"] = VARIANT
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import bench  # noqa: E402
import row_bound_coarse as rbc  # noqa: E402
import row_bound_direct as rd  # noqa: E402
import row_bound_lowrank as rl  # noqa: E402
import row_bound_model as rb  # noqa: E402

args = argparse.Namespace(impl="b200", n=a.n, dim=768, nq=a.nq, dist="latent", topk=10, gt_queries=500)
cx = bench.Ctx(args)
jv, VSF = cx.jv, cx.VSF
w = bench.World2(cx)
s = jv.GraphSearcher(w.gi)

fd, path = tempfile.mkstemp(suffix=".rbs")
os.close(fd)
os.environ["JV_ROW_BOUND_STATS_OUT"] = path
r = s.search(w.vec, w.queries, VSF.DOT_PRODUCT, 10, 100)
del os.environ["JV_ROW_BOUND_STATS_OUT"]

# one record per launch (the first pass and any retry of overflowed queries): u64 scored, dropped, drop samples, row samples; drop
# samples of 16 B, then row samples of 24 B
scored = dropped = 0
samples, row_samples = [], []
raw = np.fromfile(path, dtype=np.uint8)
os.unlink(path)
off = 0
while off < raw.size:
    c = raw[off:off + 32].view(np.uint64)
    scored, dropped = scored + int(c[0]), dropped + int(c[1])
    off += 32
    k, kr = int(c[2]), int(c[3])
    samples.append(raw[off:off + 16 * k].view(np.dtype([("q", "<i4"), ("row", "<i4"), ("last_key", "<i8")])))
    off += 16 * k
    row_samples.append(raw[off:off + 24 * kr].view(np.dtype([("q", "<i4"), ("row", "<i4"), ("last_key", "<i8"), ("key", "<i8")])))
    off += 24 * kr
smp, rsmp = np.concatenate(samples), np.concatenate(row_samples)
rs = np.random.default_rng(bench.SEED)
if smp.size > a.max_samples:
    smp = smp[np.sort(rs.choice(smp.size, a.max_samples, replace=False))]
if rsmp.size > a.max_samples:
    rsmp = rsmp[np.sort(rs.choice(rsmp.size, a.max_samples, replace=False))]
f = dropped / max(scored, 1)

import torch  # noqa: E402

rows = w.base_dev[torch.from_numpy(smp["row"].astype(np.int64)).cuda()].cpu().numpy()
qs = w.queries[smp["q"]]
d = rows.shape[1]
stride = (d + 3) & ~3
out = {"scored_rows": scored, "dropped_rows": dropped, "f": f, "samples": int(smp.size), "visited_per_query": r.visitedCount / a.nq,
       "row_bytes": 4 * stride + 8, "formats": {}}
for name, enc, sketch_bytes in (("fp16", rb.encode_fp16, 2 * stride), ("int8", rb.encode_int8, stride)):
    y, scale, rad = enc(rows, stride)
    ub = rb.dot_score_up(rb.upper_bound_raw(qs, y, scale, rad, stride))
    caught = rb.topk_key(ub, smp["row"]) < smp["last_key"]
    b = float(caught.mean())
    pred = sketch_bytes + 8 + (1.0 - f * b) * 4 * stride
    out["formats"][name] = {"b": b, "sketch_bytes": sketch_bytes, "predicted_bytes_per_row": pred, "vs_today": pred / (4 * stride + 8),
                            "median_radius_over_norm": float(np.median(rad / np.maximum(np.linalg.norm(rows, axis=1), 1e-30)))}
# the two-tier int8 sketch: the coarse half (high nibbles, c1 = 16 (c >> 4) + 8, radius r1) first, the int8 bound for what it keeps
# (scale and caught are the int8 pass of the loop above)
ss = rbc.sketch_stride(stride)
c1, _, rad1 = rbc.encode_coarse(rows, stride)
caught1 = rb.topk_key(rb.dot_score_up(rbc.upper_bound_raw(qs, c1, scale, rad1, stride)), smp["row"]) < smp["last_key"]
b, b1, b12 = out["formats"]["int8"]["b"], float(caught1.mean()), float((caught1 | caught).mean())
today = ss + 8 + 8 + (1.0 - f * b) * 4 * stride
two = (ss / 2 + 16) + 8 + (1.0 - f * b1) * ss / 2 + (1.0 - f * b12) * 4 * stride
out["int8_two_tier"] = {"b1": b1, "b12": b12, "b": b, "bytes_per_row_today": today, "predicted_bytes_per_row": two, "vs_today": two / today,
                        "median_coarse_radius_over_norm": float(np.median(rad1 / np.maximum(np.linalg.norm(rows, axis=1), 1e-30)))}
# the low-rank edge bound: settled at gather time from the expanded node's record; the others read the sketch as today
deg = w.gi.info()["degree"]
new_per_hop = r.visitedCount / max(r.expandedCountBaseLayer, 1)
xs = w.base_dev[torch.from_numpy(rl.sample_rows(a.n, a.basis_rows)).cuda()].cpu().numpy()
out["lowrank"] = {"degree": deg, "visited_per_expanded_base": new_per_hop, "bytes_per_row_today": today, "ranks": {}}
for k in (int(v) for v in a.ranks.split(",")):
    B = rl.basis(xs, k)
    codes, t, rho, beta, xn = rl.encode_rows(rows, B)
    ubl = rl.upper_bound_raw(qs, B, codes, t, rho, beta, xn, stride)
    caughtl = rb.topk_key(rb.dot_score_up(ubl), smp["row"]) < smp["last_key"]
    b1l = float(caughtl.mean())
    rec = deg * (k + 16) / new_per_hop
    pred = rec + (1.0 - f * b1l) * (ss + 16) + (1.0 - f * b) * 4 * stride
    _, _, sig, _ = rl.prepare_query(qs[:2000], B)
    out["lowrank"]["ranks"][str(k)] = {"b1": b1l, "b1_not_caught_by_int8": float((caughtl & ~caught).mean()), "record_bytes_per_new_row": rec,
                                       "predicted_bytes_per_row": pred, "vs_today": pred / today, "median_rho": float(np.median(rho)),
                                       "median_sigma": float(np.median(sig)), "median_beta": float(np.median(beta))}
# the edge tier's routing, replayed over the row samples with the k = 32 basis (the device's LR_K)
B = rl.basis(xs, rl.LR_K)
rrows = w.base_dev[torch.from_numpy(rsmp["row"].astype(np.int64)).cuda()].cpu().numpy()
rqs = w.queries[rsmp["q"]]
codes, t, rho, beta, xn = rl.encode_rows(rrows, B)
settled = rb.topk_key(rb.dot_score_up(rl.upper_bound_raw(rqs, B, codes, t, rho, beta, xn, stride)), rsmp["row"]) < rsmp["last_key"]
y8, s8, r8 = rb.encode_int8(rrows, stride)
sketch_caught = rb.topk_key(rb.dot_score_up(rb.upper_bound_raw(rqs, y8, s8, r8, stride)), rsmp["row"]) < rsmp["last_key"]
entrant = rsmp["key"] >= rsmp["last_key"]
est = ((np.float32(1) + rd.point_estimate(rqs, B, codes, t)) / np.float32(2)).astype(np.float32)


def key_score(k):
    """the score of a top-k key (the inverse of floatToSortableInt on its high word)"""
    b = np.asarray(k, dtype=np.int64) >> 32
    return np.where(b < 0, b ^ 0x7fffffff, b).astype(np.int32).view(np.float32)


cut = key_score(rsmp["last_key"])
err = est.astype(np.float64) - key_score(rsmp["key"]).astype(np.float64)
rec = deg * (rl.LR_K + 16) / new_per_hop
row_b, sk_b = 4 * stride, ss + 16
today_cost = np.where(settled, 0.0, sk_b + np.where(sketch_caught, 0.0, row_b))
bytes_today = rec + float(today_cost.mean())
lead = ~settled
out["edge_direct"] = {"row_samples": int(rsmp.size), "settled_by_edge_bound": float(settled.mean()), "entrants": float(entrant.mean()),
                      "entrants_not_settled_by_sketch": float((entrant & ~sketch_caught).mean() / max(entrant.mean(), 1e-30)),
                      "point_estimate_error_score_units": {q_: float(np.quantile(err[lead], q_)) for q_ in (0.01, 0.1, 0.5, 0.9, 0.99)},
                      "bytes_per_scored_row_today": bytes_today, "deltas": {}}
for dl in (float(v) for v in a.deltas.split(",")):
    direct = lead & (est > (cut + np.float32(dl)).astype(np.float32))
    cost = np.where(settled, 0.0, np.where(direct, row_b, sk_b + np.where(sketch_caught, 0.0, row_b)))
    pred = rec + float(cost.mean())
    out["edge_direct"]["deltas"][str(dl)] = {"entrants_routed_direct": float((direct & entrant).sum() / max(entrant.sum(), 1)),
                                             "drops_routed_direct_per_scored_row": float((direct & ~entrant).mean()),
                                             "routed_direct_per_scored_row": float(direct.mean()),
                                             "predicted_bytes_per_scored_row": pred, "vs_today": pred / bytes_today}
print(json.dumps(out, indent=1))
if a.out:
    os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
    with open(a.out, "w") as fh:
        json.dump(out, fh, indent=1)
