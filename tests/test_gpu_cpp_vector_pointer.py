"""Runs tests/cpp/test_vector_pointer.cpp on the GPU, with two slices on one device (the reference fixture's duplicated
queue) and with one: the reference's nbody and manual_stencil cases of tests/vector_pointer.cpp, a raw_pointer of a
two-part vector, which throws, and a rotation through a pointer into the target."""
import os
import subprocess
from pathlib import Path

import pytest

pytestmark = pytest.mark.gpu
BIN = Path(__file__).resolve().parent / "cpp" / "bin"


@pytest.mark.parametrize("parts", ["2", "1"])
def test_cpp_vector_pointer(built, parts):
    from vexcl_b200 import build
    build.build_cpp_tests()
    exe = BIN / "test_vector_pointer"
    assert exe.exists(), f"{exe} was not built"
    r = subprocess.run([str(exe), "12345"], capture_output=True, text=True, env=dict(os.environ, VEXCL_TEST_PARTS=parts), timeout=300)
    print(r.stdout[-3000:])
    print(r.stderr[-3000:])
    assert r.returncode == 0 and " 0 failures" in r.stdout, f"exit status {r.returncode}:\n{r.stdout[-2000:]}\n{r.stderr[-2000:]}"
