"""CPU: argument checks of ofk_gemm_bf16_grouped's output row map, before any device is touched.

The grouped output map is a TMA tensor map of whole groups (columns, rows in group, groups), so M must be a multiple
of rows_per_group.  Every rows_per_group that satisfies it is accepted: multiples of 64, divisors of 64 (one row per
group when decoding) and any other count (a prompt of arbitrary length).  Calls run in a child process with no CUDA
device visible and made-up, never dereferenced device addresses: a call that passes validation reaches device
discovery and returns OFK_ERR_CUDA."""
import json
import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ARG, NO_DEVICE = -1, -3
STORE_BF16, STORE_F32, BIAS_BF16 = 0, 1, 3
A_PTR, B_PTR, OUT_PTR, BIAS_PTR = (k << 32 for k in range(1, 5))
N, K = 128, 64


def grouped(epi, M, rpg, gs, go):
    a = dict(epi=epi, a_mn=0, b_mn=0, A=A_PTR, lda=K, B=B_PTR, ldb=K, M=M, N=N, K=K, splits=1, block_n=0, out=OUT_PTR,
             ldo=N, bias=BIAS_PTR if epi == BIAS_BF16 else 0, out_rpg=rpg, out_gs=gs, out_go=go, ak_rpg=0, ak_gs=0,
             ak_go=0, stream=0)
    return list(a.values())


CASES = {}
for epi in (STORE_BF16, STORE_F32, BIAS_BF16):
    for M, rpg in ((128, 64), (256, 128), (24, 1), (96, 8), (64, 32), (200, 100), (126, 7), (2825 * 4, 2825)):
        CASES[f"epi{epi}-M{M}-rpg{rpg}"] = (grouped(epi, M, rpg, rpg + 8, 8), NO_DEVICE)
    for M, rpg in ((130, 64), (25, 2), (100, 8), (201, 100), (127, 7)):
        CASES[f"epi{epi}-M{M}-rpg{rpg}-partial-group"] = (grouped(epi, M, rpg, rpg + 8, 8), ARG)

CHILD = r"""
import json, sys
sys.path.insert(0, sys.argv[1])
from open_flamingo_b200 import _lib
lib = _lib.lib()
cases = json.load(sys.stdin)
print(json.dumps({name: lib.ofk_gemm_bf16_grouped(*args) for name, (args, _) in cases.items()}))
"""


@pytest.fixture(scope="module")
def results():
    import __graft_entry__ as g
    g.build()
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="")
    cmd = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + ["-c", CHILD, ROOT]
    r = subprocess.run(cmd, input=json.dumps(CASES), capture_output=True, text=True, env=env, timeout=600)
    assert r.returncode == 0, r.stderr
    return json.loads(r.stdout.strip().splitlines()[-1])


@pytest.mark.parametrize("case", sorted(CASES))
def test_grouped_out_map_needs_whole_groups(results, case):
    assert results[case] == CASES[case][1], f"{case}: return code {results[case]}, expected {CASES[case][1]}"
