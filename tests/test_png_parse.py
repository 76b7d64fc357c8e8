"""b200timg_png_parse (host only) against the reference's STB source: EINVAL only where the source fails, the geometry
of every file it decodes, the APNG flag and the files the device leaves to the CPU."""
import pytest

import png_cases as pc
import timg_b200
from oracle import png as W

ref = pytest.importorskip("oracle.gif")


def test_parse_matches_pins():
    for name, data, sha, status, supported in pc.golden():
        try:
            info = timg_b200.png_parse(data)
        except timg_b200.B200Error:
            assert status == 0 and not supported, name
            continue
        assert info["supported"] == supported, (name, info["reason"])


def test_parse_matches_reference():
    if not ref.have_ref():
        pytest.skip("the reference's STB source is not built (oracle/gif.mk)")
    for name, data, sha, status, supported in pc.golden():
        r = ref.ref_stb_gif(data)
        want = None if r is None else r[0][0]
        try:
            info = timg_b200.png_parse(data)
        except timg_b200.B200Error:
            assert want is None, f"{name}: EINVAL but the reference decodes it"
            continue
        if want is not None:
            assert (info["h"], info["w"]) == want.shape[:2], name


@pytest.mark.parametrize("data", [b"", b"\x89PNG\r\n\x1a", b"GIF89a", b"\xff\xd8\xff\xd9", W.SIG, W.SIG + W.ihdr(1, 1, 8, 0)])
def test_header_failures_are_einval(data):
    with pytest.raises(timg_b200.B200Error):
        timg_b200.png_parse(data)


def test_fields_reported():
    g = {n: d for n, d in pc.golden_cases()}
    info = timg_b200.png_parse(g["trns_pal_full_il"])
    assert (info["w"], info["h"], info["bit_depth"], info["color_type"], info["interlace"]) == (12, 6, 4, 3, 1)
    assert info["palette_len"] == 16 and info["trns"] == 1 and not info["cgbi"] and not info["apng"]
    assert timg_b200.png_parse(g["trns_rgb16"])["trns"] == 2
    assert timg_b200.png_parse(g["cgbi"])["cgbi"]
    assert timg_b200.png_parse(g["apng"])["apng"] and timg_b200.png_parse(g["apng"])["supported"]
    info = timg_b200.png_parse(g["idat0_1_5"])
    assert info["idat_bytes"] > 0 and info["supported"] and info["reason"] == ""


def test_apng_rule_reads_only_the_first_kibibyte():
    s = W.samples(4, 4, 2, 8)
    late = W.png(s, 8, 2, before_idat=[(b"tEXt", bytes(1100)), (b"acTL", bytes(8))])
    assert not timg_b200.png_parse(late)["apng"]


def test_huge_skipped_chunk_is_left_to_the_cpu():
    s = W.samples(4, 4, 2, 8)
    data = W.png(s, 8, 2)
    i = data.index(b"IDAT") - 4
    bad = data[:i] + (0x80000000).to_bytes(4, "big") + b"tEXt" + data[i:]
    info = timg_b200.png_parse(bad)
    assert not info["supported"] and "2^31" in info["reason"]
