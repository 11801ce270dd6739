"""The replay recorder's kernels must not spill on sm_90a: they run inside the step loop, and a local-memory round trip
per agent row would be paid on every recorded step.  magent_b200/build.py keeps the ptxas report of backend_cuda.cu
next to the object; this test reads it (test_render_spills_cpu.function_properties parses it)."""
import os

import pytest

from magent_b200 import build as b
from test_render_spills_cpu import LOG, function_properties

KERNELS = ["replay_events_kernel", "replay_restore_kernel", "replay_record_kernel"]


@pytest.fixture(scope="module")
def report():
    if not os.path.exists(b.NVCC):
        pytest.skip("nvcc not found at " + b.NVCC)
    b.build(force=not os.path.exists(LOG))
    return function_properties(open(LOG).read())


@pytest.mark.parametrize("kernel", KERNELS)
def test_replay_kernel_has_no_spills(report, kernel):
    prefix = "_ZN2mg2be%d%sE" % (len(kernel), kernel)
    found = {name: props for name, props in report.items() if name.startswith(prefix)}
    assert len(found) == 1, "expected one %s, found %s" % (kernel, sorted(found))
    for name, props in found.items():
        assert props == (0, 0, 0), "%s: %d B stack, %d B spill stores, %d B spill loads" % ((name,) + props)
