"""CPU: the point kernel's wgmma batches run asynchronously in the built library.

A layer issues its MMAs as one batch (one commit, one wait).  If the compiler has to move accumulator registers in the
middle of a batch, ptxas injects a warpgroup.arrive there and serialises every wgmma of the function: each HGMMA then
carries its own gsb0 and is followed by its own WARPGROUP.DEPBAR, and the layer becomes a chain of single-MMA round
trips (ptxas reports C7520 / C7519).  tc::wgmma_fence_operand keeps this from happening; this test reads the SASS of
every point_kernel_pm3 instantiation and of the tensor-core self-test and checks that no HGMMA is waited for on its own.
Needs cuobjdump (CUDA toolkit), no GPU."""
import os
import re
import shutil
import subprocess

import pytest

from neuray_b200 import _lib


def _cuobjdump():
    found = shutil.which("cuobjdump")
    if found:
        return found
    for home in (os.environ.get("CUDA_HOME"), os.environ.get("CUDA_PATH"), "/usr/local/cuda"):
        if home and os.path.exists(os.path.join(home, "bin", "cuobjdump")):
            return os.path.join(home, "bin", "cuobjdump")
    return None


@pytest.fixture(scope="module")
def sass():
    tool = _cuobjdump()
    if tool is None:
        pytest.skip("cuobjdump (CUDA toolkit) not found: cannot read the library's SASS")
    assert os.path.exists(_lib.LIB_PATH), f"{_lib.LIB_PATH} not built (python -m neuray_b200.build)"
    out = subprocess.run([tool, "-sass", _lib.LIB_PATH], check=True, capture_output=True, text=True).stdout
    funcs, name = {}, None
    for line in out.splitlines():
        m = re.match(r"\s*Function : (\S+)", line)
        if m:
            name = m.group(1)
            funcs[name] = []
        elif name is not None and ("HGMMA" in line or "WARPGROUP.DEPBAR" in line):
            funcs[name].append(line)
    return funcs


def _batches(lines):
    """HGMMA lines grouped by the WARPGROUP.DEPBAR that waits for them."""
    batches, cur = [], []
    for line in lines:
        if "WARPGROUP.DEPBAR" in line:
            if cur:
                batches.append(cur)
            cur = []
        else:
            cur.append(line)
    if cur:
        batches.append(cur)
    return batches


def _check(name, lines):
    hgmma = [ln for ln in lines if "HGMMA" in ln]
    depbar = len(lines) - len(hgmma)
    assert hgmma, f"{name}: no HGMMA"
    # every batch of a layer has at least 6 MMAs (3 passes x 2 row halves); a serialised function has one DEPBAR each
    assert depbar * 4 <= len(hgmma), f"{name}: {depbar} WARPGROUP.DEPBAR for {len(hgmma)} HGMMA (wgmma serialised)"
    for i, batch in enumerate(_batches(lines)):
        gsb = [j for j, ln in enumerate(batch) if "gsb0" in ln.split(";")[0]]
        assert len(batch) >= 2 and gsb == [len(batch) - 1], (
            f"{name}: batch {i} has {len(batch)} HGMMA, gsb0 on {gsb} (only the last one may carry it)")


def test_point_kernels_issue_whole_batches(sass):
    names = [n for n in sass if "point_kernel_pm3" in n]
    assert len(names) == 14, names          # G in {4, 5, 6, 8, 10, 16, 32} x {release, DEBUG}
    for n in names:
        _check(n, sass[n])


def test_tc_selftest_issues_whole_batches(sass):
    names = [n for n in sass if "tc_selftest_kernel" in n]
    assert names
    for n in names:
        _check(n, sass[n])
