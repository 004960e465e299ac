"""GPU parity tests of the kernel / host-path VARIANTS that round 1 had written but not measured and round 2 measured,
promoted and turned on by default: the paired visited test-and-set and the
shared-memory visited set of the latency-mode kernel, 8 lanes per long L2 row, the tiled exact scan, the single-stream host
path for small batches, the batch clamp of the exact parallel build.  Every variant is exercised with its flag forced ON and
(tests/test_capi_emulated.py::test_flags_off_give_the_same_results, and the A/B tools) OFF; results must equal the oracle's
either way.  tests/test_capi_emulated.py reuses the bodies below on the emulated library in the CPU suite."""
import numpy as np
import pytest

import test_gpu_parity as G
from test_gpu_parity import SEARCH_CFGS, BIND_CFGS, METRICS, _data, kernel_mode

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def pg():
    import pg_embedding_b200 as pg
    from pg_embedding_b200 import _lib, build
    build.build()
    if pg.device_count() < 1:
        pytest.fail("no CUDA device: the product path has no CPU fallback")
    return pg


@pytest.mark.parametrize("flags", [{"PGEMB_VISITED_PAIRS": "1"}, {"PGEMB_SMEM_VISITED": "4096"}, {"PGEMB_VISITED_PAIRS": "1", "PGEMB_SMEM_VISITED": "1024"}],
                         ids=["pairs", "smem-visited", "both"])
@pytest.mark.parametrize("cfg", [SEARCH_CFGS[0], SEARCH_CFGS[5], SEARCH_CFGS[6], SEARCH_CFGS[7]], ids=lambda c: f"d{c[0]}m{c[1]}")
def test_visited_pairs_mode(pg, oracle_mod, cfg, flags, monkeypatch):
    """PGEMB_VISITED_PAIRS=1: both 32-id halves of a link list are test-and-set concurrently.  Same results, same
    traversal counters; a graph whose lists repeat an id must be detected and served by the ordered path."""
    for k, v in flags.items():
        monkeypatch.setenv(k, v)
    dims, m, efc, n, kw, efs = cfg
    rng = np.random.default_rng(4242 + dims)
    x = _data(rng, n, dims, **kw)
    q = _data(rng, 200, dims, **{k: v for k, v in kw.items() if k == "levels"})
    orc = oracle_mod.FlatIndex("port", dims, m, efc, 64, "l2", capacity=n)
    orc.build(x)
    links = orc.links()
    for dup in (False, True):
        if dup:
            # repeat an id inside the lists of a few well-connected nodes (positions in different 32-id halves when possible)
            for node in np.argsort(-links[:, 0].astype(np.int64))[:5]:
                c = int(links[node, 0])
                if c >= 2:
                    links[node, c] = links[node, 1]
            orc.set_links(links)
        idx = pg.HnswIndex(dims, m, efc, 64, "l2", capacity=n)
        idx.append(x, None, links)
        for coop, nq in (("1", 64), ("0", 200)):
            with kernel_mode(coop):
                out = idx.search_batch(q[:nq], efs[-1], want_stats=True)
            want = orc.search_many(q[:nq], efs[-1], want_counters=True)
            assert out["labels"].tobytes() == want["labels"].tobytes(), (dup, coop)
            assert out["stats"][:, :3].tolist() == want["counters"][:, :3].tolist(), (dup, coop)
        idx.close()


def test_l2_eight_lanes_per_row(pg, oracle_mod, monkeypatch):
    """PGEMB_L2_TPR8=1: long L2 rows scored by 8 lanes per row, rings of 4 rows."""
    monkeypatch.setenv("PGEMB_L2_TPR8", "1")
    monkeypatch.setenv("PGEMB_L2_TPR8_MIN_BYTES", "0")
    for cfg in (SEARCH_CFGS[3], SEARCH_CFGS[4], SEARCH_CFGS[7]):
        G.test_search_identical_to_oracle(pg, oracle_mod, "l2", cfg)
    G.test_bind_links_identical_to_oracle(pg, oracle_mod, "l2", BIND_CFGS[4])


@pytest.mark.parametrize("metric", METRICS)
def test_scan_topk_tiled(pg, oracle_mod, metric, monkeypatch):
    """The exact scan's distance step through scan_tile_kernel (rows staged once per query tile), tensor-core filter off."""
    monkeypatch.setenv("PGEMB_SCAN_TILED", "1")
    monkeypatch.setenv("PGEMB_SCAN_TC", "0")
    G.test_scan_topk_matches_exact_order(pg, oracle_mod, metric)
    G.test_scan_topk_regress_seqscan(pg)


def test_fast_small_batches_and_exact_build_clamp(pg, oracle_mod, monkeypatch):
    """PGEMB_FAST_SMALL=1 (single-stream host path for <= 64 queries, cached launch configuration) and
    PGEMB_EXACT_CLAMP_SMS=1 (exact parallel build keeps its batches at one search per SM): same results."""
    monkeypatch.setenv("PGEMB_FAST_SMALL", "1")
    for case in G.GOLD:
        G.test_kat_regress(pg, case)
    rng = np.random.default_rng(77)
    n, dims, m, efc = 4000, 48, 8, 40
    x = _data(rng, n, dims)
    q = _data(rng, 100, dims)
    orc = oracle_mod.FlatIndex("port", dims, m, efc, 64, "l2", capacity=n)
    orc.build(x)
    idx = pg.HnswIndex(dims, m, efc, 64, "l2", capacity=n)
    idx.append(x, orc.labels(), orc.links())
    for nq, ef in ((1, 10), (1, 10), (64, 16), (100, 16), (3, 40), (1, 64)):
        out = idx.search_batch(q[:nq], ef, want_stats=True)
        want = orc.search_many(q[:nq], ef, want_counters=True)
        assert out["labels"].tobytes() == want["labels"].tobytes() and out["stats"][:, :3].tolist() == want["counters"][:, :3].tolist(), (nq, ef)
    assert idx.search(q[0], 12).tolist() == orc.search(q[0], 12).tolist()
    idx.close()
    monkeypatch.setenv("PGEMB_EXACT_CLAMP_SMS", "1")
    idx = pg.HnswIndex(dims, m, efc, 64, "l2", capacity=n)
    idx.append(x)
    idx.build_exact(0, n, 1024)
    assert idx.links().tobytes() == orc.links().tobytes()
    idx.close()

