"""The oracle's model of the bulk build (`FlatIndex.build_bulk`: `oracle_bind_batch` driven by `bulk_schedule`), which
tests/test_gpu_bulk_build.py holds pgemb_build_bulk to byte for byte.  Here, without a GPU: its schedule is capi.cu's, one
node per batch is the sequential build that tests/test_oracle_vs_ref.py pins to the compiled reference, and with larger
batches it builds another graph on the data of the GPU and emulated cases -- so their comparison is not vacuous."""
import pytest

from test_gpu_bulk_build import CASES, EMU_CASES, case_data


def test_schedule(oracle_mod):
    s = oracle_mod.bulk_schedule
    # node 0 is skipped, batches tile the rest, one node at a time until 64 are bound
    sched = s(0, 200_000, 4096)
    assert sched[0] == (1, 1) and sched[62] == (63, 1) and sched[63] == (64, 2)
    assert all(p + b == q for (p, b), (q, _) in zip(sched, sched[1:])) and sum(b for _, b in sched) == 199_999
    # a batch is pos / 32 nodes: the bench's cap of 4096 applies only from node 131 072 on
    assert all(b == min(p // 32, 4096, 200_000 - p) or b == 1 for p, b in sched)
    capped = [p for p, b in sched if b == 4096]
    assert capped and min(capped) >= 131_072 and all(b < 4096 for p, b in sched if p < 131_072)
    # first > 0 starts at first / 32; batch_max is clamped to [1, 65536]
    assert s(1000, 100, 4096)[0] == (1000, 31) and s(0, 1, 64) == []
    assert s(0, 500, 0) == s(0, 500, 1) == [(p, 1) for p in range(1, 500)]
    big = s(0, 3_000_000, 1 << 20)
    assert max(b for _, b in big) == 1 << 16 and big == s(0, 3_000_000, 1 << 16)


def test_ref_has_no_model(oracle_mod):
    if not oracle_mod.available("ref"):
        pytest.skip("the compiled reference is not built here")
    with pytest.raises(ValueError):
        oracle_mod.FlatIndex("ref", 4, 2, 8, 8, "l2", capacity=4).build_bulk(0, 4, 8)


def _model(oracle_mod, cfg, batch_max, seq_prefix=0):
    name, metric, dims, m, efc, n, kw = cfg
    x, _, labels = case_data(cfg)
    idx = oracle_mod.FlatIndex("port", dims, m, efc, 64, metric, capacity=n)
    if seq_prefix:
        idx.build(x[:seq_prefix], labels[:seq_prefix])
    idx.append_unbound(x[seq_prefix:], labels[seq_prefix:])
    idx.build_bulk(seq_prefix, n - seq_prefix, batch_max)
    return idx


def _sequential(oracle_mod, cfg):
    name, metric, dims, m, efc, n, kw = cfg
    x, _, labels = case_data(cfg)
    idx = oracle_mod.FlatIndex("port", dims, m, efc, 64, metric, capacity=n)
    idx.build(x, labels)
    return idx


@pytest.mark.parametrize("cfg", EMU_CASES + CASES[3:4] + CASES[10:11], ids=lambda c: c[0])
def test_one_node_batches_are_the_sequential_build(oracle_mod, cfg):
    seq = _sequential(oracle_mod, cfg).links()
    assert _model(oracle_mod, cfg, 1).links().tobytes() == seq.tobytes()
    assert _model(oracle_mod, cfg, 1, seq_prefix=cfg[5] // 3).links().tobytes() == seq.tobytes()


@pytest.mark.parametrize("cfg", EMU_CASES + CASES, ids=lambda c: c[0])
def test_batches_change_the_graph(oracle_mod, cfg):
    """Every case with m > 0 differs from the sequential build at each batch_max > 1 it runs with (with m = 0 there are no
    links to differ: that case pins that the build runs at all)."""
    seq = _sequential(oracle_mod, cfg).links()
    for bmax in ((8, 64) if cfg in EMU_CASES else (8, 64, 4096)):
        differ = int((_model(oracle_mod, cfg, bmax).links() != seq).any(1).sum())
        if cfg[3] == 0:
            assert differ == 0 and not seq.any()
        else:
            assert differ > 0, (cfg[0], bmax)
