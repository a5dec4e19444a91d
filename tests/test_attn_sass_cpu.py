"""CPU tests on the wgmma attention kernel as built (no GPU needed).

Inside a consumer, Q K^T of tile j and P V of tile j - 1 are issued together and wgmma_wait<1> retires only Q K^T, so the
softmax of tile j can run while P V is on the tensor cores.  That only happens if ptxas leaves the softmax between the
two waits; it is free to move the full wait up (it did, until the wait got a basic block of its own), so the SASS is
checked here.
"""
import os
import re

from tests.test_attention_tc_gpu import BKV, STAGES
from tests.test_sass_cpu import _sass_functions
from videoswap_b200 import _lib

SRC = os.path.join(os.path.dirname(_lib.LIB_PATH), "csrc", "attention_tc.cu")


def test_softmax_runs_under_pv():
    funcs = {n: body for n, body in _sass_functions(_lib.LIB_PATH).items() if "attn_tc_kernel" in n}
    assert len(funcs) == 2, f"expected the d = 40 and d = 80 attention kernels, found {sorted(funcs)}"
    for name, body in funcs.items():
        between, inside = [], None
        for line in body:
            m = re.search(r"WARPGROUP\.DEPBAR\.LE\s+gsb0,\s*0x(\d)", line)
            if m:
                if inside is not None:
                    between.append(inside)
                inside = 0 if m.group(1) == "1" else None
            elif inside is not None and "MUFU.EX2" in line:
                inside += 1
        assert between, f"{name}: no wgmma_wait<1> followed by wgmma_wait<0>"
        # one exp2 per score (BKV / 2 per thread) plus the two rescale factors
        assert max(between) >= BKV // 2, f"{name}: only {max(between)} MUFU.EX2 between wgmma_wait<1> and <0>"


def test_edge_shapes_follow_tile_config():
    """The GPU edge-case shapes in test_attention_tc_gpu.py are built from the kernel's key tile and ring depth."""
    src = open(SRC).read()
    assert re.search(r"static constexpr int BKV = (\d+);", src).group(1) == str(BKV)
    m = re.search(r"static constexpr int STAGES = D > 64 \? (\d+) : (\d+);", src)
    assert m and (int(m.group(2)), int(m.group(1))) == (STAGES[40], STAGES[80])
