"""C++-level drop-in check on the GPU: oracle/_ref/adapter_check links the reference's own objects, the
adapters of timg_b200/csrc/adapters.h and libb200timg.so, and drives the reference canvases/scaler and
ours through the SAME interfaces (ImageScaler, TerminalCanvas + BufferedWriteSequencer), comparing the
bytes that reach the file descriptor.  The sixel canvas has no linkable reference counterpart (libsixel
is not in the tree): its in-tree framing (src/sixel-canvas.cc:100-155) is checked byte for byte around the
library's own DCS stream."""
import os
import subprocess

import pytest

pytestmark = pytest.mark.gpu
BIN = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "oracle", "_ref", "adapter_check")


@pytest.mark.skipif(not os.path.exists(BIN), reason="oracle/_ref/adapter_check not built (needs the reference's sources)")
def test_cpp_adapters_produce_reference_bytes():
    r = subprocess.run([BIN], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "ADAPTER CHECK OK" in r.stdout and "DIFFERENT" not in r.stdout
