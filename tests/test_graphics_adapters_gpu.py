"""C++-level drop-in check of the kitty / iTerm2 adapters on the GPU: oracle/_ref/graphics_adapter_check
(oracle/graphics.mk) links the reference's own KittyGraphicsCanvas / ITerm2GraphicsCanvas, compiled with a
stored-block compressor in place of libdeflate, the adapters of timg_b200/csrc/adapters.h and libb200timg.so, and
drives both through the same TerminalCanvas + BufferedWriteSequencer, comparing the bytes that reach the file
descriptor (kitty's time-seeded image ids normalised)."""
import os
import subprocess

import pytest

pytestmark = pytest.mark.gpu

BIN = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "oracle", "_ref", "graphics_adapter_check")


@pytest.mark.skipif(not os.path.exists(BIN), reason="oracle/_ref/graphics_adapter_check not built (needs the reference's sources)")
def test_kitty_and_iterm2_adapters_produce_reference_bytes():
    r = subprocess.run([BIN], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "GRAPHICS ADAPTER CHECK OK" in r.stdout and "DIFFERENT" not in r.stdout
    assert r.stdout.count("identical") == 4
