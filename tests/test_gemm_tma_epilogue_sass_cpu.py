"""CPU: static checks on the GEMM epilogue of the shipped libofk.so (cuobjdump -sass, no GPU needed).

Every GEMM kernel writes its outputs with asynchronous TMA stores from a shared-memory epilogue buffer
(cp.async.bulk.tensor, UTMASTG in SASS), so none issues a per-thread global store.  The ATOMIC_F32 kernels add into
their output with a TMA reduce (cp.reduce.async.bulk.tensor...add, UTMAREDG...ADD) and issue no per-thread global
reduction (RED / REDG), which keeps exactly one fp32 add per element per launch."""
import re
import shutil
import subprocess

import pytest

ATOMIC_F32 = 2   # OFK_EPI_ATOMIC_F32 (include/ofk.h)


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


def epilogue_of(kernel_name):
    """The EPI template argument of a mangled gemm_kernel<A_MN, B_MN, EPI> name."""
    m = re.search(r"gemm_kernelILi([01])ELi([01])ELi(\d+)E", kernel_name)
    assert m, kernel_name
    return int(m.group(3))


def test_every_gemm_kernel_stores_through_tma(gemm_sass):
    for k, ops_ in gemm_sass.items():
        if epilogue_of(k) == ATOMIC_F32:
            continue
        assert any(o.startswith("UTMASTG") for o in ops_), f"{k}: no TMA store"


def test_gemm_kernels_issue_no_per_thread_global_stores(gemm_sass):
    for k, ops_ in gemm_sass.items():
        st = sorted({o for o in ops_ if o.split(".")[0] in ("STG", "ST")})
        assert not st, f"{k}: per-thread global stores {st}"


def test_atomic_kernels_reduce_through_tma_only(gemm_sass):
    atomic = {k: v for k, v in gemm_sass.items() if epilogue_of(k) == ATOMIC_F32}
    assert len(atomic) == 4
    for k, ops_ in atomic.items():
        assert any(o.startswith("UTMAREDG") and ".ADD" in o for o in ops_), f"{k}: no TMA reduce-add"
        red = sorted({o for o in ops_ if o.split(".")[0] in ("RED", "REDG", "ATOM", "ATOMG")})
        assert not red, f"{k}: per-thread global reductions {red}"
