"""A stream-ordered BQ top-k (jv_topk_bruteforce_device_async) still running on the caller's stream must not share device scratch
with a host-pointer search that the same thread issues meanwhile: that search takes the overlap path (queries streamed on a second
stream behind an arrival watermark), and each of the two keeps its own buffers in the thread's context. Both results must equal
the same calls run on their own, bit for bit."""
import ctypes as C

import numpy as np
import pytest

import oracle_lib as o

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def jv():
    import jvector_b200
    jvector_b200.init()
    return jvector_b200


@pytest.fixture(scope="module")
def lib(jv):
    from jvector_b200 import _native
    return _native.load()


def test_async_bq_topk_and_overlapped_search_keep_their_own_scratch(jv, lib):
    import torch

    from jvector_b200 import _native as nat
    rng = np.random.default_rng(11)
    dim = 768
    # BQ rows the tensor-core contraction takes: 768 / 64 = 12 words (even), n >= 4096
    bq_rows = rng.standard_normal((20000, dim)).astype(np.float32)
    bq = jv.BQVectors(jv.bq_encode_all(bq_rows), dim)
    tq = rng.standard_normal((512, dim)).astype(np.float32)
    k = 64
    _, _, want_keys = jv.topk_bruteforce(bq, o.COSINE, tq, k)

    # a graph to search with 400 host queries at dim 768 (1.2 MB): large enough for the overlapped copy
    data = o.random_unit_vectors(rng, 6000, dim)
    vec = jv.F32Vectors(data)
    gi = jv.GraphIndexBuilder(jv.VectorSimilarityFunction.DOT_PRODUCT, M=16, beamWidth=60).build(vec)
    sq = o.random_unit_vectors(rng, 400, dim)
    assert sq.nbytes >= 1 << 20
    searcher = jv.GraphSearcher(gi)
    alone = searcher.search(vec, sq, jv.VectorSimilarityFunction.DOT_PRODUCT, 10, 40)

    qd = torch.from_numpy(tq).cuda()
    keys = torch.empty((len(tq), k), dtype=torch.int64, device="cuda")
    status = torch.full((1,), -7, dtype=torch.int32, device="cuda")
    stream = torch.cuda.Stream()
    torch.cuda.synchronize()
    nat.check(lib.jv_topk_bruteforce_device_async(bq._h, o.COSINE, C.c_void_p(qd.data_ptr()), len(tq), k, 0, C.c_void_p(keys.data_ptr()),
                                                  C.c_void_p(status.data_ptr()), C.c_void_p(stream.cuda_stream)))
    # no synchronisation of `stream`: the top-k may still be running while this search stages its queries and watermark
    during = searcher.search(vec, sq, jv.VectorSimilarityFunction.DOT_PRODUCT, 10, 40)
    torch.cuda.synchronize()

    assert int(status.item()) == 0
    assert np.array_equal(keys.cpu().numpy(), want_keys)
    assert np.array_equal(during.nodes, alone.nodes)
    assert np.array_equal(np.asarray(during.scores).view(np.int32), np.asarray(alone.scores).view(np.int32))
    gi.close()
    vec.close()
    bq.close()
