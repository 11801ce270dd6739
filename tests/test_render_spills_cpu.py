"""The small-view observation render must not spill on sm_90a.

The render is a store stream at 64 registers per thread (32 warps per SM); local-memory spills inside its tile loop
compete with the plane reads for L1 and with the output for L2.  magent_b200/build.py keeps the ptxas report of
backend_cuda.cu next to the object; this test reads it."""
import os
import re

import pytest

from magent_b200 import build as b

LOG = os.path.join(b.HERE, "lib", "backend_cuda_cu.o.ptxas.log")

# obs_render_kernel<T, NIT = 4, TURN = false, TA>, every tile width TA: float (the reference ABI, the battle
# workloads) and __half
SPILL_FREE = {"obs_render_kernel<float, 4, false, TA>": "_ZN2mg2be17obs_render_kernelIfLi4ELb0ELi",
              "obs_render_kernel<__half, 4, false, TA>": "_ZN2mg2be17obs_render_kernelI6__halfLi4ELb0ELi"}


def function_properties(text):
    """{mangled name: (stack frame, spill store, spill load bytes)} of every sm_90a entry in a ptxas -v report"""
    pat = re.compile(r"Function properties for (\S+)\n\s+(\d+) bytes stack frame, (\d+) bytes spill stores, "
                     r"(\d+) bytes spill loads")
    return {m.group(1): tuple(int(m.group(i)) for i in (2, 3, 4)) for m in pat.finditer(text)}


@pytest.fixture(scope="module")
def report():
    if not os.path.exists(b.NVCC):
        pytest.skip("nvcc not found at " + b.NVCC)
    b.build(force=not os.path.exists(LOG))
    return function_properties(open(LOG).read())


@pytest.mark.parametrize("kernel", sorted(SPILL_FREE))
def test_small_view_render_has_no_spills(report, kernel):
    found = {name: props for name, props in report.items() if name.startswith(SPILL_FREE[kernel])}
    assert len(found) == 2, "expected a narrow and a wide tile of %s, found %s" % (kernel, sorted(found))
    for name, props in found.items():
        assert props == (0, 0, 0), "%s: %d B stack, %d B spill stores, %d B spill loads" % ((name,) + props)
