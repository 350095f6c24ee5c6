"""CPU: static checks on the GEMM kernels of the shipped libofk.so (cuobjdump -sass, no GPU needed).

A wide tile keeps 128 fp32 accumulators per consumer thread; a register spill would show up as local-memory traffic
(LDL / STL) in the mainloop or the epilogue.  Every instantiation can run the 2-CTA clustered tile, so every one must
load its share of B with a multicast TMA load."""
import re
import shutil
import subprocess

import pytest


@pytest.fixture(scope="module")
def gemm_sass():
    if shutil.which("cuobjdump") is None:
        pytest.skip("cuobjdump not on PATH")
    import __graft_entry__ as g
    g.build()
    from open_flamingo_b200 import _lib
    out = subprocess.run(["cuobjdump", "-sass", _lib.LIB_PATH], capture_output=True, text=True, check=True).stdout
    kernels, name = {}, None
    for line in out.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            name = m.group(1)
            kernels[name] = []
        elif name is not None:
            m = re.search(r"^\s+/\*[0-9a-f]+\*/\s+(?:@!?U?P\d+\s+)?([A-Z][A-Z0-9_.]*)", line)
            if m:
                kernels[name].append(m.group(1))
    gemms = {k: v for k, v in kernels.items() if "gemm_kernel" in k}
    assert len(gemms) == 10 * 4
    return gemms


def test_gemm_kernels_have_no_local_memory_traffic(gemm_sass):
    for k, ops_ in gemm_sass.items():
        local = sorted({o for o in ops_ if o.split(".")[0] in ("LDL", "STL")})
        assert not local, f"{k}: local-memory instructions {local}"


def test_gemm_kernels_multicast_the_shared_operand(gemm_sass):
    for k, ops_ in gemm_sass.items():
        assert "UTMALDG.2D.MULTICAST" in ops_, f"{k}: no multicast TMA load"
        assert "UTMALDG.2D" in ops_, f"{k}: no per-CTA TMA load"
