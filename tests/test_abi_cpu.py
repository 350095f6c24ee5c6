"""CPU: libofk.so loads and exports exactly the entry points include/ofk.h declares (no compute calls here)."""
import ctypes
import os
import re

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def header_functions():
    src = open(os.path.join(ROOT, "include", "ofk.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(ofk_[a-z0-9_]+)\s*\(", src)))


def test_library_exports_every_declared_symbol():
    import __graft_entry__ as g
    g.build()  # nvcc cross-compiles for sm_90a without a GPU
    from open_flamingo_b200 import _lib
    lib = ctypes.CDLL(_lib.LIB_PATH)
    declared = header_functions()
    assert declared, "no declarations parsed from include/ofk.h"
    for name in declared:
        assert hasattr(lib, name), f"{name} declared in ofk.h but not exported by libofk.so"
    assert sorted(_lib.exported_symbols()) == declared, "ctypes signature table and ofk.h disagree"
    loaded = _lib.lib()
    assert loaded.ofk_abi_version() == 4
    assert isinstance(_lib.launch_count(), int)


def test_no_cpu_fallback():
    """The product path must fail loudly off-GPU rather than silently computing on the CPU."""
    import pytest
    import torch
    from open_flamingo_b200 import ops
    from open_flamingo_b200.src.helpers import GatedCrossAttentionBlock, PerceiverResampler
    with pytest.raises(RuntimeError):
        ops.gemm(torch.zeros(16, 16, dtype=torch.bfloat16), torch.zeros(16, 16, dtype=torch.bfloat16))
    with pytest.raises(RuntimeError):
        PerceiverResampler(dim=64, depth=1)(torch.zeros(1, 1, 1, 4, 64))
    with pytest.raises(RuntimeError):
        GatedCrossAttentionBlock(dim=64, dim_visual=64)(torch.zeros(1, 4, 64), torch.zeros(1, 1, 64, 64),
                                                        media_locations=torch.zeros(1, 4, dtype=torch.bool))


def test_product_never_imports_oracle():
    pkg = os.path.join(ROOT, "open_flamingo_b200")
    for dirpath, _, files in os.walk(pkg):
        for f in files:
            if f.endswith(".py"):
                text = open(os.path.join(dirpath, f)).read()
                assert "oracle" not in text.replace("# oracle", ""), f"{f} references the oracle"


def _sass_by_kernel():
    import shutil
    import subprocess
    import pytest
    if shutil.which("cuobjdump") is None:
        pytest.skip("cuobjdump not on PATH")
    from open_flamingo_b200 import _lib
    out = subprocess.run(["cuobjdump", "-sass", _lib.LIB_PATH], capture_output=True, text=True, check=True).stdout
    kernels, name = {}, None
    for line in out.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            name = m.group(1)
            kernels[name] = set()
        elif name is not None:
            m = re.search(r"^\s+/\*[0-9a-f]+\*/\s+(?:@!?U?P\d+\s+)?([A-Z][A-Z0-9_]*)", line)
            if m:
                kernels[name].add(m.group(1))
    return kernels


def test_hot_kernels_are_wgmma_and_tma_in_the_shipped_binary():
    """Static proof, on the .so the tests load: every GEMM kernel issues warpgroup MMAs (HGMMA) on operands staged by TMA
    (UTMALDG), with no mma.sync (HMMA) path inside; every attention core issues wgmma and no mma.sync."""
    kernels = _sass_by_kernel()
    assert len(kernels) > 40
    gemms = {k: v for k, v in kernels.items() if "gemm_kernel" in k}
    assert len(gemms) == 10 * 4   # epilogues x A/B operand layouts
    for k, ops_ in gemms.items():
        assert "HGMMA" in ops_, f"{k}: no wgmma"
        assert "UTMALDG" in ops_, f"{k}: operands are not staged by TMA"
        assert "HMMA" not in ops_, f"{k}: mma.sync inside a wgmma kernel"
    attn = {k: v for k, v in kernels.items() if re.search(r"attn_fwd_kernel|attn_bwd_dq_kernel|attn_bwd_dkv_kernel|"
                                                          r"dense\d+fwd_kernel|dense\d+bwd_dq_kernel|dense\d+bwd_dkv_kernel", k)}
    assert len(attn) == 3 + 3 * 2, sorted(attn)   # media cores + dense cores for head_dim 64 and 128
    for k, ops_ in attn.items():
        assert "HGMMA" in ops_, f"{k}: attention core without wgmma"
        assert "HMMA" not in ops_, f"{k}: mma.sync inside a wgmma attention core"
