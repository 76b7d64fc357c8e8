"""C++-level drop-in check of the kitty / iTerm2 adapters with deflate = true on the GPU:
oracle/_ref/graphics_deflate_adapter_check (oracle/graphics_deflate.mk) links the reference's own KittyGraphicsCanvas
(plain and tmux form) and ITerm2GraphicsCanvas, compiled with a libdeflate stand-in that replays given zlib streams,
B200KittyCanvas / B200ITerm2Canvas (timg_b200/csrc/adapters.h) and libb200timg.so.  Each adapter runs first; the
reference canvas then runs over the same frames with the adapter's own zlib streams, and the bytes that reach the file
descriptors must be identical.  The binary pins time(), so both sides pick the same image ids, and stubs system()."""
import os
import subprocess

import pytest

pytestmark = pytest.mark.gpu

BIN = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "oracle", "_ref",
                   "graphics_deflate_adapter_check")


@pytest.mark.skipif(not os.path.exists(BIN), reason="oracle/_ref/graphics_deflate_adapter_check not built (needs the reference's sources)")
def test_deflate_adapters_produce_reference_bytes_around_their_streams():
    r = subprocess.run([BIN], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "GRAPHICS DEFLATE ADAPTER CHECK OK" in r.stdout and "DIFFERENT" not in r.stdout
    assert r.stdout.count("identical") == 6 and r.stdout.count("stored bytes compressed") == 6
