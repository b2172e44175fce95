"""CPU: the kernels' dynamic shared-memory limit, carveout and occupancy are set and read in one
place, smem_optin (csrc/api.cu).  The limit is per-device state and the occupancy depends on each
launch's shared memory; a kernel that opts in calls the helper rather than keeping its own copy."""
import glob
import os
import re

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "yet_another_mobilenet_series_b200", "csrc")
HELPER = "api.cu"
NAMES = ("cudaFuncAttributeMaxDynamicSharedMemorySize",
         "cudaFuncAttributePreferredSharedMemoryCarveout",
         "cudaOccupancyMaxActiveBlocksPerMultiprocessor")


def _sources():
    paths = [p for ext in ("*.cu", "*.cuh", "*.h") for p in glob.glob(os.path.join(CSRC, ext))]
    assert len(paths) > 10, paths
    return paths


def test_only_the_helper_sets_shared_memory_attributes():
    found = []
    for path in _sources():
        if os.path.basename(path) == HELPER:
            continue
        with open(path) as f:
            for n, line in enumerate(f, 1):
                found += ["%s:%d: %s" % (os.path.basename(path), n, name)
                          for name in NAMES if name in line]
    assert not found, "call smem_optin (csrc/host_util.h) instead:\n" + "\n".join(found)


def test_helper_defines_them():
    with open(os.path.join(CSRC, HELPER)) as f:
        src = f.read()
    assert re.search(r"^int smem_optin\(", src, re.M)
    for name in NAMES:
        assert name in src, name
