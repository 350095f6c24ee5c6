"""CPU: static checks on the attention cores of the shipped libofk.so (cuobjdump -sass, no GPU needed).

The cores double-buffer their K/V (or Q/dO) tiles; a stage chosen by the loop index must be an address computed from
it, not a pointer read from a local array, which costs local-memory stores and loads (STL / LDL) in every kernel."""
import re
import shutil
import subprocess

import pytest

ATTN = re.compile(r"attn_fwd_kernel|attn_bwd_dq_kernel|attn_bwd_dkv_kernel|delta_kernel|"
                  r"dense\d+fwd_kernel|dense\d+bwd_dq_kernel|dense\d+bwd_dkv_kernel")


@pytest.fixture(scope="module")
def attn_sass():
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
    attn = {k: v for k, v in kernels.items() if ATTN.search(k)}
    assert len(attn) == 3 + 3 * 2 + 2   # media cores, dense cores at head_dim 64 and 128, delta at 64 and 128
    return attn


def test_attention_kernels_have_no_local_memory_traffic(attn_sass):
    for k, ops_ in attn_sass.items():
        local = sorted({o for o in ops_ if o.split(".")[0] in ("LDL", "STL")})
        assert not local, f"{k}: local-memory instructions {local}"
