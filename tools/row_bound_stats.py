#!/usr/bin/env python
"""How many bytes a row sketch would save the c2 walk: builds the c2 world the way bench.py does (1M x 768 latent rows, 10 000
queries, DOT_PRODUCT, topK 10, rerankK 100), runs one search on a counter build of the library (-DJV_ROW_BOUND_STATS, built here
with tools/build_variant.sh) and reports

    f = share of the level-0 rows the walk scores that JV_EMIT drops against a full candidate list,
    b = share of those drops that the sketch's upper bound (tests/row_bound_model.py) still catches,

for the fp16 sketch and for an int8 sketch with one scale per row; b is replayed on the host over a sample of the drops
({query, row, key of the list's last entry}). Predicted bytes per visited row = sketch + 8 + (1 - f b) 4 d, against 4 d + 8.

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
ap.add_argument("--out", default="")
a = ap.parse_args()

if not os.path.exists(VARIANT):
    subprocess.run([os.path.join(ROOT, "tools", "build_variant.sh"), "rbs", "-DJV_ROW_BOUND_STATS"], check=True, stdout=subprocess.DEVNULL)
os.environ["JV_B200_SO"] = VARIANT
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import bench  # noqa: E402
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

# one record per launch (the first pass and any retry of overflowed queries): u64 scored, dropped, samples; samples of 16 B
scored = dropped = 0
samples = []
raw = np.fromfile(path, dtype=np.uint8)
os.unlink(path)
off = 0
while off < raw.size:
    c = raw[off:off + 24].view(np.uint64)
    scored, dropped = scored + int(c[0]), dropped + int(c[1])
    off += 24
    k = int(c[2])
    samples.append(raw[off:off + 16 * k].view(np.dtype([("q", "<i4"), ("row", "<i4"), ("last_key", "<i8")])))
    off += 16 * k
smp = np.concatenate(samples)
rs = np.random.default_rng(bench.SEED)
if smp.size > a.max_samples:
    smp = smp[np.sort(rs.choice(smp.size, a.max_samples, replace=False))]
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
print(json.dumps(out, indent=1))
if a.out:
    os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
    with open(a.out, "w") as fh:
        json.dump(out, fh, indent=1)
