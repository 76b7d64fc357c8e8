"""C++-level drop-in check of kitty's tmux form on the GPU: oracle/_ref/kitty_tmux_adapter_check (oracle/graphics_tmux.mk)
links the reference's own KittyGraphicsCanvas, compiled with a stored-block compressor in place of libdeflate,
B200KittyCanvas (timg_b200/csrc/adapters.h) and libb200timg.so, drives both with tmux_passthrough_needed = true
through the same TerminalCanvas + BufferedWriteSequencer and compares the bytes that reach the file descriptor.  The
binary pins time(), so both sides pick the same image ids, and records system(), so each side's one
"tmux set -p allow-passthrough on" is checked and no shell runs."""
import os
import subprocess

import pytest

pytestmark = pytest.mark.gpu

BIN = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "oracle", "_ref", "kitty_tmux_adapter_check")


@pytest.mark.skipif(not os.path.exists(BIN), reason="oracle/_ref/kitty_tmux_adapter_check not built (needs the reference's sources)")
def test_kitty_tmux_adapter_produces_reference_bytes():
    r = subprocess.run([BIN], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "KITTY TMUX ADAPTER CHECK OK" in r.stdout and "DIFFERENT" not in r.stdout and "WRONG" not in r.stdout
    assert r.stdout.count("identical, passthrough command once on each side") == 4
