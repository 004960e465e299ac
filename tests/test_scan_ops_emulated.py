"""pgemb_scan_topk_op on the host-emulated library (capi.cu compiled by g++, its kernels run by tests/emu's SIMT emulator):
the exact scan under any of the three operators over a mirror of any metric, on the exact kernels (PGEMB_SCAN_TC=0) and
on the tensor-core filter's orchestration and re-scoring (=2; the wgmma product itself is a host stand-in).  The bodies are
tests/test_gpu_scan_ops.py's, at small sizes."""
import ctypes as C

import numpy as np
import pytest

import test_gpu_scan_ops as S

pytestmark = pytest.mark.timeout(1800, method="thread")


@pytest.fixture(scope="module")
def emu_lib(tmp_path_factory):
    from emu_build import build_emulated
    from pg_embedding_b200 import _lib
    return _lib._bind(C.CDLL(build_emulated(tmp_path_factory.mktemp("emu_scan_ops"))))


@pytest.fixture()
def pg(emu_lib, monkeypatch):
    """pg_embedding_b200 with its library handle swapped for the emulated build (restored after each test)."""
    import pg_embedding_b200 as pkg
    from pg_embedding_b200 import _lib
    monkeypatch.setattr(_lib, "_lib", emu_lib)
    monkeypatch.setenv("PGEMB_EMU_SMS", "2")
    monkeypatch.setenv("PGEMB_EMU_TMA", "late")
    assert pkg.device_count() == 1
    return pkg


@pytest.mark.parametrize("shape", [(300, 19, 6, 9), (200, 8, 4, 256)], ids=["n300d19k9", "n200d8k256"])
def test_nine_pairs_match_the_oracle(pg, oracle_mod, monkeypatch, shape):
    """All 3 x 3 (mirror, query) metric pairs, both paths, every query against the oracle: deleted rows, a tie, a zero row and a
    zero query (cosine NaN), 19 dims (padded rows); k = 256 above the 181 live rows of the second table."""
    n, dims, nq, k = shape
    S.check_pairs(pg, oracle_mod, monkeypatch, n, dims, nq, k, range(nq))


@pytest.mark.parametrize("tc_first", ["0", "2"])
def test_l2_mirror_computes_norms_on_demand(pg, oracle_mod, monkeypatch, tc_first):
    S.check_norms_on_demand(pg, oracle_mod, monkeypatch, 240, 13, 5, 6, tc_first)


@pytest.mark.parametrize("metric", ["l2", "cosine", "manhattan"])
def test_zero_rows(pg, monkeypatch, metric):
    """An empty mirror and one whose rows are all deleted: no results under any operator, tails (~0, +inf)."""
    for tc in ("0", "2"):
        monkeypatch.setenv("PGEMB_SCAN_TC", tc)
        for deleted in (None, True):
            idx = pg.HnswIndex(6, 3, 8, 4, metric, capacity=8)
            if deleted:
                idx.append(np.ones((5, 6), np.float32), np.arange(5, dtype=np.uint64) | S.DELETED)
            for op in S.METRICS:
                got = idx.scan_topk(np.ones((2, 6), np.float32), 3, metric=op)
                assert got["n"].tolist() == [0, 0]
                assert (got["labels"] == np.uint64(0xFFFFFFFFFFFFFFFF)).all() and np.isinf(got["dists"]).all()
            idx.close()


def test_own_metric_gives_pgemb_scan_topk_bytes_and_counters(pg, monkeypatch):
    """pgemb_scan_topk is pgemb_scan_topk_op with the mirror's metric: the same bytes and the same counter deltas."""
    rng = np.random.default_rng(5)
    n, dims, nq, k = 260, 12, 7, 8
    x, q, labels = S.table(rng, n, dims, nq)
    for metric in S.METRICS:
        idx = pg.HnswIndex(dims, 4, 8, 16, metric, capacity=n)
        idx.append(x, labels)
        for tc in ("0", "1", "2"):
            monkeypatch.setenv("PGEMB_SCAN_TC", tc)
            c0 = S.counters()
            own = idx.scan_topk(q, k)
            c1 = S.counters()
            named = idx.scan_topk(q, k, metric=metric)
            c2 = S.counters()
            for f in ("labels", "dists", "n"):
                assert own[f].tobytes() == named[f].tobytes(), (metric, tc, f)
            assert S.delta(c0, c1) == S.delta(c1, c2), (metric, tc)
        idx.close()


def test_device_entry_point_and_bad_metrics(pg):
    """pgemb_scan_topk_op_device (all memory is host memory here) == pgemb_scan_topk_op; metrics outside 0 .. 2 are refused
    by both entry points with PGEMB_ERR_ARG, as is a null index."""
    from pg_embedding_b200 import _lib
    lib = _lib.load()
    rng = np.random.default_rng(6)
    n, dims, nq, k = 90, 7, 3, 5
    x, q, labels = S.table(rng, n, dims, nq)
    idx = pg.HnswIndex(dims, 4, 8, 16, "cosine", capacity=n)
    idx.append(x, labels)
    vp = lambda a: a.ctypes.data_as(C.c_void_p)
    for mi, metric in enumerate(S.METRICS):
        ol, od, on = np.zeros((nq, k), np.uint64), np.zeros((nq, k), np.float32), np.zeros(nq, np.int32)
        _lib.check(lib.pgemb_scan_topk_op_device(idx.dev, mi, nq, vp(q), k, vp(ol), vp(od), vp(on), None))
        host = idx.scan_topk(q, k, metric=metric)
        assert ol.tobytes() == host["labels"].tobytes() and od.tobytes() == host["dists"].tobytes() and on.tolist() == host["n"].tolist()
    f32p, u64p, i32p = C.POINTER(C.c_float), C.POINTER(C.c_uint64), C.POINTER(C.c_int32)
    for bad in (-1, 3, 1 << 30):
        assert lib.pgemb_scan_topk_op(idx.dev, bad, nq, q.ctypes.data_as(f32p), k, ol.ctypes.data_as(u64p), None, on.ctypes.data_as(i32p)) == 2
        assert b"unknown distance function" in lib.pgemb_last_error()
        assert lib.pgemb_scan_topk_op_device(idx.dev, bad, nq, vp(q), k, vp(ol), None, vp(on), None) == 2
    assert lib.pgemb_scan_topk_op(None, 0, nq, q.ctypes.data_as(f32p), k, ol.ctypes.data_as(u64p), None, on.ctypes.data_as(i32p)) == 2
    with pytest.raises(KeyError):
        idx.scan_topk(q, k, metric="hamming")
    idx.close()
