"""No C++ exception crosses the C ABI: a host allocation that fails inside an entry point comes back as GB_ERR_CAPACITY
with gb_last_error() naming it, and the calling process lives on."""
import subprocess
import sys
from pathlib import Path

import pytest

ROOT = Path(__file__).resolve().parent.parent

# Runs in its own process, so the lowered address-space limit cannot reach the test runner.  With
# mapping_cap_per_read = 2^32 - 1, the first training window of gb_map_paired_job sizes a host std::vector of
# 2 reads x (2^32 - 1) mappings x 8 bytes = 64 GiB before any CUDA call; RLIMIT_AS refuses that reservation outright,
# whatever the overcommit setting, so nothing is ever touched.  The limit is restored before the device is closed.
CHILD = r"""
import ctypes as C, resource, sys
sys.path.insert(0, sys.argv[1])
import numpy as np
from vg_b200 import capi, synth

index = synth.make_tiny_graph().build_index()
dev = capi.Device(index, 0)
dist = capi.FragmentDistribution()
p = capi.default_map_params()
p.mapping_cap_per_read = 0xffffffff
reads = np.frombuffer(b"ACGT" * 75, dtype=np.uint8).copy()
read_off = np.array([0, 150, 300], dtype=np.uint64)
aln, status = np.zeros(2, dtype=capi.alignment_dt), np.zeros(2, dtype=np.uint8)
maps, edits, route = np.zeros(1, dtype=capi.mapping_dt), np.zeros(1, dtype=np.uint32), np.zeros(1, dtype=np.uint8)
used = (C.c_uint64(), C.c_uint64())
lib = capi.load_library()

vm_kib = next(int(line.split()[1]) for line in open("/proc/self/status") if line.startswith("VmSize:"))
soft, hard = resource.getrlimit(resource.RLIMIT_AS)
resource.setrlimit(resource.RLIMIT_AS, (vm_kib * 1024 + (1 << 30), hard))
rc = lib.gb_map_paired_job(dev.handle, C.byref(p), dist._h, 0, 2, capi.ptr(reads), None, capi.ptr(read_off), capi.ptr(aln),
                           capi.ptr(maps), len(maps), capi.ptr(edits), len(edits), capi.ptr(status), capi.ptr(route),
                           C.byref(used[0]), C.byref(used[1]))
message = lib.gb_last_error().decode()
resource.setrlimit(resource.RLIMIT_AS, (soft, hard))
assert rc == capi.GB_ERR_CAPACITY, (rc, message)
assert "out of host memory" in message, message
dev.close()
print("status", rc, message)
"""


@pytest.mark.gpu
def test_host_allocation_failure_is_a_status_code():
    run = subprocess.run([sys.executable, "-c", CHILD, str(ROOT)], capture_output=True, text=True, timeout=600)
    assert run.returncode == 0, run.stdout + run.stderr
    assert "status -4 gb_map_paired_job: out of host memory" in run.stdout, run.stdout
