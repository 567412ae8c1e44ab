"""searcher.search(&query, &(Count, TopDocs)) through the C++ host mirror: tests/cpp/host_mirror_count_tests.cpp, built by
`make -C tantivy_b200/csrc` next to the library.  Each half of the pair must equal what its collector alone returns."""
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BIN = os.path.join(ROOT, "tantivy_b200", "_lib", "host_mirror_count_tests")


def test_binary_is_built():
    assert os.access(BIN, os.X_OK), f"{BIN} is missing: build with `make -C tantivy_b200/csrc`"


@pytest.mark.gpu
def test_count_and_top_docs_through_the_host_mirror():
    r = subprocess.run([BIN], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "0 test(s) failed" in r.stdout and r.stdout.count("ok  ") == 2, r.stdout
