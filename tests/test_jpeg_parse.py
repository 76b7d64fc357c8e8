"""b200timg_jpeg_parse (host only) against the reference's STB source: EINVAL only where the source fails, the
geometry of every file it decodes, and the files the device leaves to the CPU."""
import pytest

import timg_b200
import jpeg_cases as jc

ref = pytest.importorskip("oracle.gif")


def _ref(data):
    if not ref.have_ref():
        pytest.skip("the reference's STB source is not built (oracle/gif.mk)")
    r = ref.ref_stb_gif(data)
    return None if r is None else r[0][0]


@pytest.mark.parametrize("name,data", jc.small_cases() + jc.surgery_cases(), ids=lambda v: v if isinstance(v, str) else "")
def test_parse_matches_reference(name, data):
    want = _ref(data)
    try:
        info = timg_b200.jpeg_parse(data)
    except timg_b200.B200Error:
        assert want is None, f"{name}: EINVAL but the reference decodes it"
        return
    if want is not None:
        assert (info["h"], info["w"]) == want.shape[:2]
    assert info["supported"], info["reason"]


def test_progressive_is_left_to_the_cpu():
    data = jc.jpeg(jc.photo(40, 30), quality=85, progressive=True)
    info = timg_b200.jpeg_parse(data)
    assert info["progressive"] and not info["supported"] and "progressive" in info["reason"]


def test_second_scan_is_left_to_the_cpu():
    base = jc.jpeg(jc.photo(40, 30), quality=85, subsampling=2)
    i = base.index(b"\xff\xda")
    twice = base[:-2] + base[i:]
    info = timg_b200.jpeg_parse(twice)
    assert not info["supported"] and "scan" in info["reason"]


@pytest.mark.parametrize("data", [b"", b"\xff\xd8", b"GIF89a", b"\xff\xd8\xff\xc0\x00\x05"])
def test_header_failures_are_einval(data):
    with pytest.raises(timg_b200.B200Error):
        timg_b200.jpeg_parse(data)


def test_sampling_and_restart_reported():
    info = timg_b200.jpeg_parse(jc.jpeg(jc.photo(70, 50), quality=85, subsampling=1, restart_marker_rows=1))
    assert info["h_samp"] == [2, 1, 1] and info["v_samp"] == [1, 1, 1] and info["restart_interval"] > 0


def test_parse_matches_pins():
    for name, data, sha, status, supported in jc.golden():
        try:
            info = timg_b200.jpeg_parse(data)
        except timg_b200.B200Error:
            assert status == 0 and not supported, name
            continue
        assert info["supported"] == supported, (name, info["reason"])
