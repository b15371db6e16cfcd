"""Where the LM loop's and the covariance pass's per-thread state lives, as ptxas reports it for sm_90a: compiles gicp.cu
with -Xptxas -v (no GPU needed) and holds the stack frame, the spill bytes and the static shared memory of the hot kernels
to the budgets of DESIGN.md §3.  A change that moves the traversal stack or the slot cache back to local memory, or adds
spills, shows up here before it shows up as time."""
import os
import re
import shutil
import subprocess

import pytest

from b200reg import build

# mangled-name fragment -> (max stack frame bytes, max spill store bytes, max spill load bytes, max static shared bytes)
BUDGETS = {
    # 1-NN walk: 6 stack entries in shared memory (6 KB), 58 deeper ones in local arrays (464 B) touched only past depth 6;
    # the slot cache is dynamic shared memory sized to the batch
    "k_gicp_search": (536, 68, 68, 6192),
    # 15-NN walk: the 15 KB result heap in shared memory, the traversal stack in local memory
    "k_covarianceILi15E": (720, 192, 200, 15360),
    # the linearize pass, spill-free at 4 blocks per SM; no static shared memory (the slot cache is dynamic)
    "k_gicp_accum": (256, 0, 0, 0),
}


def _nvcc():
    return build.NVCC if os.path.exists(build.NVCC) else shutil.which("nvcc")


@pytest.fixture(scope="module")
def ptxas_report(tmp_path_factory):
    nvcc = _nvcc()
    if not nvcc:
        pytest.skip("nvcc not available")
    out = tmp_path_factory.mktemp("ptxas") / "gicp.o"
    cmd = [nvcc] + build.FLAGS + ["-Xptxas", "-v", "-c", os.path.join(build.CSRC, "gicp.cu"), "-o", str(out)]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    kernels = {}
    name = None
    for line in r.stderr.splitlines():
        m = re.search(r"Compiling entry function '(\w+)' for 'sm_90a'", line)
        if m:
            name = m.group(1)
            kernels[name] = {"smem": 0}
            continue
        if name is None:
            continue
        m = re.search(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", line)
        if m:
            kernels[name].update(frame=int(m.group(1)), st=int(m.group(2)), ld=int(m.group(3)))
        m = re.search(r"Used (\d+) registers.*?(?:(\d+) bytes smem)?$", line)
        if m:
            kernels[name]["regs"] = int(m.group(1))
            if m.group(2):
                kernels[name]["smem"] = int(m.group(2))
    return kernels


@pytest.mark.parametrize("kernel", sorted(BUDGETS))
def test_kernel_state_within_budget(ptxas_report, kernel):
    hits = [k for k in ptxas_report if kernel in k]
    assert len(hits) == 1, (kernel, sorted(ptxas_report))
    got = ptxas_report[hits[0]]
    frame, st, ld, smem = BUDGETS[kernel]
    assert got["frame"] <= frame, got
    assert got["st"] <= st and got["ld"] <= ld, got
    assert got["smem"] <= smem, got
