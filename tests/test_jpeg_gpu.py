"""b200timg_jpeg_frames on the GPU, what is particular to JPEG: the segment sweep one file at a time, sized files and
the rejections of files the device does not take.  test_decode_gpu.py holds what JPEG shares with PNG."""
import hashlib

import pytest

import jpeg_cases as jc
import timg_b200
from test_decode_gpu import check

pytestmark = pytest.mark.gpu


def test_review_case_and_sweep_each_alone(ctx):
    """Segments of 1, 2 and 3 mod 64 bytes: the last subsequence starts after the marker was reached."""
    for name, data, sha, want, _ in jc.golden():
        if name.startswith(("seg_", "sweep")):
            canv, status = ctx.jpeg_frames([data])
            assert int(status[0]) == want == 1
            assert hashlib.sha256(canv[0].tobytes()).hexdigest() == sha, name


@pytest.mark.parametrize("k", range(5))
def test_sized(ctx, k):
    name, data = jc.sized_cases()[k]
    canv, status = ctx.jpeg_frames([data])
    check(name, data, canv[0], int(status[0]))


def test_rejections_launch_nothing(ctx):
    good = jc.jpeg(jc.photo(16, 16), quality=85)
    prog = jc.jpeg(jc.photo(16, 16), quality=85, progressive=True)
    l0 = ctx.launches
    with pytest.raises(timg_b200.B200Error, match="file 1"):
        ctx.jpeg_frames([good, prog])
    with pytest.raises(timg_b200.B200Error):
        ctx.jpeg_frames([b"\xff\xd8\xff\xd9"])
    assert ctx.launches == l0
