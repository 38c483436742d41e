"""Runs tests/cpp/test_scan.cpp on the GPU, with two slices on one device (the reference fixture's duplicated queue)
and with one: the reference's scan.cpp (inclusive, exclusive), scan_by_key.cpp (sbk) and reduce_by_key.cpp (rbk)
cases, sort_by_key followed by reduce_by_key against a host group-by, init counted once across parts, and the
refusals."""
import os
import subprocess
from pathlib import Path

import pytest

pytestmark = pytest.mark.gpu
BIN = Path(__file__).resolve().parent / "cpp" / "bin"


@pytest.mark.parametrize("parts", ["2", "1"])
def test_cpp_scan(built, parts):
    from vexcl_b200 import build
    build.build_cpp_tests()
    exe = BIN / "test_scan"
    assert exe.exists(), f"{exe} was not built"
    r = subprocess.run([str(exe), "12345"], capture_output=True, text=True, env=dict(os.environ, VEXCL_TEST_PARTS=parts), timeout=300)
    print(r.stdout[-3000:])
    print(r.stderr[-3000:])
    assert r.returncode == 0 and " 0 failures" in r.stdout, f"exit status {r.returncode}:\n{r.stdout[-2000:]}\n{r.stderr[-2000:]}"
