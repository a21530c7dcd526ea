"""K_fused8 keeps everything in registers: ptxas's report for both instantiations (depth and multidepth) shows no spill.
A spill puts local-memory traffic into every tile of the packed8 reduce.  Reads the log `make` writes next to depth.o."""
import os
import re

import pytest

LOG = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "build", "depth.ptxas.log")


def test_fused8_has_no_spills():
    if not os.path.exists(LOG):
        pytest.skip("no ptxas log: the library was not built here")
    text = open(LOG).read()
    found = {}
    for m in re.finditer(r"Compiling entry function '(\S*depth_fused8_kernel\S*)'[^\n]*\n(.*?)\n(.*?)\n", text):
        spill = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", m.group(2) + m.group(3))
        assert spill, m.group(0)
        found[m.group(1)] = (int(spill.group(1)), int(spill.group(2)))
    assert len(found) == 2, found
    assert all(v == (0, 0) for v in found.values()), found
