"""make_search_config (csrc/search_config.h): the shared-memory layout the traversal kernel is launched with, over a grid of
shapes (dims 1..2000, maxM 0..200, ef 1..4000, both kernel modes, 4 and 8 lanes per row).  A layout mistake shows up on
the GPU only as a misaligned-address fault or silent corruption, so the invariants the kernel relies on are checked here:
size within a CTA's 227 KB, 16-byte alignment of everything a bulk copy or a vector load touches, 8-byte alignment of
64-bit keys and mbarriers, regions inside their block and not overlapping, sane ring / slot counts."""
import csv
import io
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def rows(tmp_path_factory):
    exe = str(tmp_path_factory.mktemp("cfg") / "config_probe")
    res = subprocess.run(["g++", "-std=c++17", "-O1", "-o", exe, os.path.join(ROOT, "tests", "cfg", "config_probe.cpp")], capture_output=True, text=True)
    assert res.returncode == 0, res.stderr
    out = subprocess.run([exe], capture_output=True, text=True, check=True).stdout
    return [{k: int(v) for k, v in r.items()} for r in csv.DictReader(io.StringIO(out))]


def test_layout_invariants(rows):
    assert len(rows) > 5000
    ok = [r for r in rows if r["rc"] == 0]
    assert len(ok) > 0.8 * len(rows)
    for r in ok:
        what = {k: r[k] for k in ("metric", "dim", "maxM", "ef", "coop", "tpr")}
        row_bytes = ((r["dim"] + 3) & ~3) * 4
        link_bytes = ((r["maxM"] + 1 + 3) & ~3) * 4
        rows_per_ring = 32 // r["tpr"]
        assert r["smem"] <= 232448, what                                     # 227 KB per CTA
        assert 1 <= r["rings"] <= 15 and 1 <= r["warps"] <= 32, what
        assert r["rings"] <= r["warps"] or r["coop"], what
        # rows land by bulk copy (16-byte aligned destination and size) and are read with vector loads
        assert r["row_smem"] % 16 == 0 and r["row_smem"] >= row_bytes, what
        assert r["ring_bytes"] % 128 == 0 and r["ring_bytes"] >= rows_per_ring * r["row_smem"], what
        assert r["off_ring"] % 128 == 0 and r["off_ring"] >= r["off_pool"] + r["pool_size"], what
        assert r["off_priv"] % 128 == 0 and r["off_priv"] >= r["off_ring"] + r["rings"] * r["ring_bytes"], what
        assert r["priv_bytes"] % 128 == 0, what
        nslots_cta = 1 if r["coop"] else r["warps"]
        assert r["off_priv"] + nslots_cta * r["priv_bytes"] <= r["smem"], what
        # inside a slot's private block
        assert r["off_qt"] % 16 == 0 and r["off_qtail"] % 16 == 0, what       # LDS.128 of the transposed query
        assert r["off_res"] % 8 == 0 and r["off_hopkey"] % 8 == 0 and r["off_acckey"] % 8 == 0 and r["off_evict"] % 8 == 0, what   # u64 keys
        assert r["off_pf"] % 16 == 0, what                                     # link row arrives by bulk copy
        assert r["off_pfbar"] % 8 == 0, what                                   # mbarrier
        assert r["off_hopid"] % 4 == 0, what
        order = ["off_qt", "off_qtail", "off_res", "off_hopkey", "off_acckey", "off_evict", "off_hopid", "off_pf", "off_pfbar"]
        offs = [r[k] for k in order]
        assert offs == sorted(offs), what
        hopcap = max(r["maxM"], 1)
        assert r["off_hopkey"] - r["off_res"] >= 2 * r["ef"] * 8, what        # two result buffers
        assert r["off_acckey"] - r["off_hopkey"] >= hopcap * 8, what
        assert r["off_pfbar"] - r["off_pf"] >= link_bytes, what
        assert r["off_pfbar"] + 8 <= r["priv_bytes"], what
        # conflict-free pitches (DESIGN.md section 6): rows == 16 (cosine/manhattan) or 32 (L2) mod 128, query runs 4 (or 2) words past a multiple of 32
        assert r["row_smem"] % 128 == (32 if r["metric"] == 0 else 16), what
        assert r["qt_stride"] % 32 == 4, what                                    # every run 16-byte aligned (LDS.128), runs on distinct banks
        # slots the host allocates per-slot workspace for
        assert r["slots"] == (132 if r["coop"] else 132 * r["warps"]), what
    # what does not fit must say so instead of producing a layout
    for r in rows:
        if r["rc"] != 0:
            assert r["rc"] in (1, 2)
    # the north-star shape keeps its measured configuration: 12 slots sharing 6 rings
    ns = [r for r in ok if (r["metric"], r["dim"], r["maxM"], r["ef"], r["coop"], r["tpr"]) == (1, 768, 64, 64, 0, 4)]
    assert len(ns) == 1 and (ns[0]["warps"], ns[0]["rings"]) == (12, 6)
