"""b200timg_qoi_parse against the pins of tests/golden/qoi.npz, the plan model of qoi_cases.py against qoi.cu's
constexprs, and each split-point case landing where its name says (no GPU)."""
import ctypes as C
import os
import re

import pytest

import qoi_cases as qc
import timg_b200
from oracle import qoi as Q

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_parse_matches_pins():
    for name, data, parse, _, _, _, _ in qc.golden():
        if parse < 0:
            with pytest.raises(timg_b200.B200Error):
                timg_b200.qoi_parse(data)
            continue
        info = timg_b200.qoi_parse(data)
        assert info["supported"], name
        assert (info["w"], info["h"]) == (int.from_bytes(data[4:8], "big"), int.from_bytes(data[8:12], "big")), name
        assert (info["channels"], info["colorspace"]) == (data[12], data[13]), name


def test_rejection_expectations_match_pins():
    pins = {g[0]: g[2] for g in qc.golden()}
    for name, _, ok in qc.rejections():
        assert (pins[name] >= 0) == ok, name


def test_files_of_2_31_bytes_are_not_taken():
    data = Q.stream(2, 2, Q.Ops().rgb(1, 2, 3))
    info = timg_b200.QoiInfo()
    for size, want in ((len(data), 1), ((1 << 31) - 1, 1), (1 << 31, 0)):
        assert timg_b200.lib().b200timg_qoi_parse(data, size, C.byref(info)) == timg_b200.OK
        assert info.supported == want, size
    assert b"int" in info.reason


def test_model_constants_match_kernels():
    src = open(os.path.join(ROOT, "timg_b200", "csrc", "qoi.cu")).read()
    for name in ("TILE", "CHUNK", "SEG", "CK", "ROUNDS"):
        m = re.search(rf"constexpr int {name} = (\d+);", src)
        assert m and int(m.group(1)) == getattr(qc, name), name
    assert "7 + ROUNDS kernels" in src


def test_split_cases_land_where_named():
    names = set()
    for name, data, where in qc.split_cases():
        assert name not in names
        names.add(name)
        ops = qc.live_ops(data)
        starts = [o for o, _ in ops]
        if "straddle" in where:
            at, boundary = where["straddle"]
            assert at in starts and at < boundary < at + qc.op_len(data[at]), name
            assert qc.tile_of(at) + 1 == qc.tile_of(boundary), name
        if "op_at" in where:
            k, first = where["op_at"]
            assert data[starts[k]] == first, name
            assert k % qc.CK in (0, 1, qc.CK - 1), name
        if "rounds" in where:
            m, slot = where["rounds"]
            assert len(ops) == (m + 1) * qc.SEG, name      # segments 0..m
            reads = [i for i, (o, _) in enumerate(ops) if data[o] == slot]
            assert reads == [m * qc.SEG], name              # the stale slot is read once, by segment m's first op
            assert m in (qc.ROUNDS - 1, qc.ROUNDS, qc.ROUNDS + 1)
        if where.get("diff_only"):
            assert all(data[o] >> 6 == 1 for o in starts[1:]), name
            assert len(ops) > 2 * qc.SEG
    straddles = {(w["straddle"][1] - w["straddle"][0]) for _, _, w in qc.split_cases() if "straddle" in w}
    assert straddles == {1, 2, 3, 4}
