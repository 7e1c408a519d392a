"""Multi-GPU plumbing (one process per GPU, torch.distributed): the ONLY exchange step of the path is the final top-k
merge (SURVEY §8e).

  * graph search (configs 2/3): every rank holds a replica of the base + graph; queries are sharded; no data-path collective.
  * brute-force first pass (config 4): the base is range-sharded by contiguous node-id range; every rank scores ALL queries
    against its shard and keeps a local top-k of 64-bit keys (reference ordering key, NodeQueue.java:125-137, node ids made
    global on the device); ONE all_gather of [nq][k] int64 per rank (NCCL over NVLink on GPUs, gloo in the CPU tests),
    then a k-way merge per query (device kernel jv_topk_merge_device; `merge_keys_host` is the host restatement the gloo
    tests use to check the plumbing without a GPU).
"""
import numpy as np


def shard_range(n, rank, world):
    """contiguous node-id range [lo, hi) of `rank` (remainder spread over the first ranks)"""
    base, rem = divmod(n, world)
    lo = rank * base + min(rank, rem)
    return lo, lo + base + (1 if rank < rem else 0)


KEY_MIN = np.iinfo(np.int64).min


def rebase_keys_host(keys, id_base):
    """node id += id_base inside a key (low word is ~node): key -= id_base, pads untouched"""
    keys = np.asarray(keys, dtype=np.int64)
    return np.where(keys == KEY_MIN, keys, keys - np.int64(id_base))


def merge_keys_host(gathered, k):
    """gathered: [world][nq][k] keys -> [nq][k] best first (host restatement of topk_merge_kernel)"""
    g = np.asarray(gathered, dtype=np.int64)
    world, nq, kk = g.shape
    allk = np.transpose(g, (1, 0, 2)).reshape(nq, world * kk)
    allk = np.sort(allk, axis=1)[:, ::-1]
    out = np.full((nq, k), KEY_MIN, dtype=np.int64)
    out[:, : min(k, allk.shape[1])] = allk[:, :k]
    return out


def keys_to_nodes_scores(keys):
    keys = np.asarray(keys, dtype=np.int64)
    nodes = ((~keys) & 0xffffffff).astype(np.int64)
    s = (keys >> 32).astype(np.int32)
    bits = (s ^ ((s >> 31) & 0x7fffffff)).astype(np.int32)
    nodes = np.where(keys == KEY_MIN, -1, nodes).astype(np.int32)
    return nodes, bits.view(np.float32)


class ShardedBruteForce:
    """Exhaustive top-k over a base range-sharded across the ranks of a torch.distributed group.

    local_topk(queries, k) -> int64 [nq][k] keys with GLOBAL node ids, as a torch tensor on this rank's device.
    The default implementation calls the C ABI (jv_topk_bruteforce_device); tests inject an oracle-backed one under gloo."""

    def __init__(self, dist, local_topk, merge=None):
        self.dist = dist
        self.local_topk = local_topk
        self.merge = merge

    def search(self, queries, k):
        import torch
        dist = self.dist
        world = dist.get_world_size() if dist is not None and dist.is_initialized() else 1
        local = self.local_topk(queries, k)
        if world == 1:
            gathered = local.unsqueeze(0)
        else:
            flat = torch.empty((world * local.shape[0], local.shape[1]), dtype=torch.int64, device=local.device)
            dist.all_gather_into_tensor(flat, local.contiguous())
            gathered = flat.view(world, local.shape[0], local.shape[1])
        if self.merge is not None:
            return self.merge(gathered, k)
        return torch.from_numpy(merge_keys_host(gathered.cpu().numpy(), k))


def gpu_sharded_bruteforce(dist, vectors, vsf, id_base):
    """ShardedBruteForce over a device-resident shard (`vectors` holds rows [id_base, id_base + n)).

    BQ shards take the stream-ordered C entry points: local top-k (tensor-core contraction), the all-gather and the merge are
    enqueued on torch's current stream with no host synchronisation; `status()` (call it after the timed region) returns the
    number of queries the device left unresolved since the last check. Other kinds use the synchronous entry points."""
    import ctypes as C

    import torch

    from . import _native as nat
    lib = nat.init()
    status = torch.zeros(2, dtype=torch.int32, device="cuda")  # [0] this step, [1] running total
    use_async = [True]

    def local_topk(queries, k):
        q = queries if isinstance(queries, torch.Tensor) else torch.from_numpy(np.ascontiguousarray(queries, dtype=np.float32)).cuda()
        q = q.contiguous()
        keys = torch.empty((q.shape[0], k), dtype=torch.int64, device=q.device)
        if use_async[0]:
            st = torch.cuda.current_stream().cuda_stream
            rc = lib.jv_topk_bruteforce_device_async(vectors._h, int(vsf), C.c_void_p(q.data_ptr()), q.shape[0], k, int(id_base), C.c_void_p(keys.data_ptr()),
                                                     C.c_void_p(status.data_ptr()), C.c_void_p(st))
            if rc == 0:
                status[1] += status[0]
                return keys
            if rc != -5:  # JV_ERR_UNSUPPORTED: not a BQ shard the contraction kernel takes
                nat.check(rc)
            use_async[0] = False
        torch.cuda.synchronize()
        nat.check(lib.jv_topk_bruteforce_device(vectors._h, int(vsf), C.c_void_p(q.data_ptr()), q.shape[0], k, int(id_base), C.c_void_p(keys.data_ptr())))
        return keys

    def merge(gathered, k):
        world, nq, kk = gathered.shape  # shard-major, as all_gather_into_tensor leaves it
        g = gathered.contiguous()
        out = torch.empty((nq, k), dtype=torch.int64, device=gathered.device)
        if kk == k:
            st = torch.cuda.current_stream().cuda_stream
            nat.check(lib.jv_topk_merge_device_async(C.c_void_p(g.data_ptr()), nq, world, kk, C.c_void_p(out.data_ptr()), C.c_void_p(st)))
            return out
        flat = g.permute(1, 0, 2).contiguous()
        torch.cuda.synchronize()
        nat.check(lib.jv_topk_merge_device(C.c_void_p(flat.data_ptr()), nq, world, kk, C.c_void_p(out.data_ptr())))
        return out

    sb = ShardedBruteForce(dist, local_topk, merge)
    sb.status = lambda: int(status[1].item())
    return sb


class SliceExchange:
    """The exchange step of the sharded build: `count` items of `width` int32 each (+ one int32 per item) are produced slice-wise —
    rank r fills positions [r * chunk, (r + 1) * chunk) with chunk = ceil(count / world) — and all-gathered so that every rank
    holds positions 0 .. count-1 in order. produce(lo, hi, rows_ptr, deg_ptr) receives pointers to a VIRTUAL [count][width] /
    [count] array of which only rows lo .. hi-1 exist (they are rows 0 .. of this rank's send buffer), which is the contract of
    jv_builder_insert_slice / jv_builder_reprune_slice."""

    def __init__(self, dist, device):
        self.dist = dist
        self.device = device
        self.world = dist.get_world_size() if dist is not None and dist.is_initialized() else 1
        self.rank = dist.get_rank() if self.world > 1 else 0
        self.bufs = {}
        self.exchanged_bytes = 0

    def _buf(self, name, rows, width):
        import torch
        t = self.bufs.get(name)
        if t is None or t.shape[0] < rows:
            t = torch.empty((max(rows, 1) + max(rows, 1) // 4, width), dtype=torch.int32, device=self.device)
            self.bufs[name] = t
        return t

    def run(self, count, width, produce):
        import ctypes as C

        from . import _native as nat
        world, rank = self.world, self.rank
        chunk = (count + world - 1) // world
        lo, hi = min(count, rank * chunk), min(count, (rank + 1) * chunk)
        send, sdeg = self._buf("send%d" % width, chunk, width), self._buf("sdeg", chunk, 1)
        nat.check(produce(lo, hi, C.c_void_p(send.data_ptr() - lo * width * 4), C.c_void_p(sdeg.data_ptr() - lo * 4)))
        if world == 1:
            return send, sdeg
        allr, alld = self._buf("all%d" % width, world * chunk, width), self._buf("alld", world * chunk, 1)
        self.dist.all_gather_into_tensor(allr[:world * chunk], send[:chunk])
        self.dist.all_gather_into_tensor(alld[:world * chunk], sdeg[:chunk])
        self.exchanged_bytes += world * chunk * (width + 1) * 4
        return allr, alld


def sharded_build(dist, vectors, vsf, M=32, beamWidth=100, neighborOverflow=1.2, alpha=1.2, addHierarchy=True, seed=0, max_batch=0, concurrent_window=-1):
    """GraphIndexBuilder.build with the insert scoring SHARDED over the ranks of `dist` (BASELINE config 5).

    Every rank holds a replica of the rows (`vectors`, resident fp32) and of the adjacency. Per batch of inserted nodes: each rank
    runs the beam searches + robust prunes of ITS slice (jv_builder_insert_slice), ONE all-gather moves the new rows, every rank
    applies the whole batch (sorted back-links: the replicas stay bit-identical), then the rows that passed overflow * M are re-pruned
    slice-wise and all-gathered the same way. NCCL calls and kernels share torch's current stream. dist = None: one rank (the
    same code path, no collective). `vectors` may be PQVectors instead (pqBuildScoreProvider: jv_builder_create_pq) or BQVectors
    (bqBuildScoreProvider: jv_builder_create_bq). Returns (GraphIndex, device_ms, exchanged_bytes)."""
    import ctypes as C

    import torch

    from . import _native as nat
    from .api import BQVectors, GraphIndex, PQVectors
    lib = nat.init()
    world = dist.get_world_size() if dist is not None and dist.is_initialized() else 1
    rank = dist.get_rank() if world > 1 else 0
    params = nat.BuildParams(M, beamWidth, neighborOverflow, alpha, 1 if addHierarchy else 0, seed, max_batch, concurrent_window)
    st = torch.cuda.current_stream().cuda_stream
    b = C.c_void_p()
    create = lib.jv_builder_create_pq if isinstance(vectors, PQVectors) else lib.jv_builder_create_bq if isinstance(vectors, BQVectors) else lib.jv_builder_create
    nat.check(create(vectors._h, int(vsf), C.byref(params), C.c_void_p(st), C.byref(b)))
    deg_, cap_, mb_ = C.c_int(), C.c_int(), C.c_int()
    nat.check(lib.jv_builder_info(b, C.byref(deg_), C.byref(cap_), C.byref(mb_)))
    degree, row_cap, mb = deg_.value, cap_.value, mb_.value
    ex = SliceExchange(dist, "cuda")

    def exchange(count, width, produce):
        return ex.run(count, width, produce)

    def reprune_round(L):
        if L <= 0:
            return
        rows, dg = exchange(L, row_cap, lambda lo, hi, rp, dp: lib.jv_builder_reprune_slice(b, lo, hi, rp, dp))
        nat.check(lib.jv_builder_apply_repruned(b, L, C.c_void_p(rows.data_ptr()), C.c_void_p(dg.data_ptr())))

    first, count, L = C.c_int32(), C.c_int32(), C.c_int32()
    try:
        while True:
            nat.check(lib.jv_builder_next_batch(b, C.byref(first), C.byref(count)))
            if count.value == 0:
                break
            f, c = first.value, count.value
            rows, dg = exchange(c, degree, lambda lo, hi, rp, dp: lib.jv_builder_insert_slice(b, f, c, lo, hi, rp, dp))
            nat.check(lib.jv_builder_apply_new(b, f, c, C.c_void_p(rows.data_ptr()), C.c_void_p(dg.data_ptr()), C.byref(L)))
            reprune_round(L.value)
        nat.check(lib.jv_builder_collect_over_degree(b, C.byref(L)))
        reprune_round(L.value)
        g = C.c_void_p()
        ms = C.c_double()
        nat.check(lib.jv_builder_finish(b, C.byref(g), C.byref(ms)))
    finally:
        lib.jv_builder_free(b)
    return GraphIndex(_handle=g), ms.value, ex.exchanged_bytes
