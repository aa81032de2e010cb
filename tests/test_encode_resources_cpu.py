"""The encode kernel's per-family instances, as compiled into the library: the Fast instance (levels 10 and 11) must stay
free of local memory within the 72 registers that 28 resident warps per SM allow, and the Generic instance (every other
level) must not grow the stack frame it had when the families were split (656 bytes).  A spill slot in the Fast parser's
hot loop goes to L2 at this residency, so a change that brings one back should fail here, before it is measured."""
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "lizard_b200", "liblizard_b200.so")
FAM_FAST, FAM_FAST_BIG, FAM_GENERIC = 0, 1, 2       # EncFamily, csrc/encode_core.cuh


def _cuobjdump():
    exe = shutil.which("cuobjdump")
    if exe is None:
        home = os.environ.get("CUDA_HOME") or os.environ.get("CUDA_PATH") or "/usr/local/cuda"
        cand = os.path.join(home, "bin", "cuobjdump")
        exe = cand if os.path.exists(cand) else None
    return exe


def _encode_instances():
    exe = _cuobjdump()
    if exe is None:
        pytest.skip("cuobjdump not available")
    out = subprocess.run([exe, "-res-usage", LIB], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True,
                         check=True).stdout
    found = {}
    name = None
    for line in out.splitlines():
        m = re.search(r"Function (\S+):", line)
        if m:
            name = m.group(1)
            continue
        if name and "REG:" in line:
            f = re.search(r"lizard_encode_units_kernelILi(\d+)E", name)
            if f:
                found[int(f.group(1))] = {k: int(v) for k, v in re.findall(r"(REG|STACK|LOCAL):(\d+)", line)}
            name = None
    return found


def test_encode_kernel_has_one_instance_per_family():
    assert sorted(_encode_instances()) == [FAM_FAST, FAM_FAST_BIG, FAM_GENERIC]


def test_fast_instance_is_spill_free():
    fast = _encode_instances()[FAM_FAST]
    assert fast["STACK"] == 0 and fast["LOCAL"] == 0, fast
    assert fast["REG"] <= 72, fast


def test_generic_instance_stack_does_not_grow():
    gen = _encode_instances()[FAM_GENERIC]
    assert gen["STACK"] <= 656, gen
    assert gen["REG"] <= 72, gen
