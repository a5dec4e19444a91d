"""CPU test on the compiled sm_90a code of the built library (no GPU needed): the short-K linears' and GEGLUs' epilogue-slot
instantiations (gemm_tc_kernel<BN, EPI, GemmParamsEpi>) read no global memory with LDG -- the producer warpgroup brings
every operand in with TMA (UTMALDG) and bulk copies (UBLKCP) and the consumers read shared memory -- and no
gemm_tc_kernel instantiation uses local memory (register spills)."""
import re
import subprocess

from tests.test_sass_cpu import _cuobjdump, _sass_functions
from videoswap_b200 import _lib


def test_slot_instantiations_issue_no_global_loads():
    funcs = {n: body for n, body in _sass_functions(_lib.LIB_PATH).items() if "gemm_tc_kernel" in n}
    slot = {n: body for n, body in funcs.items() if "GemmParamsEpi" in n}
    # BLOCK_N 128 and 160 x RES, LNOUT, LNOUT + RES, LN, LN + RV; BLOCK_N 256 x GEGLU, GEGLU + LN
    assert len(slot) == 12, sorted(slot)
    for n, body in slot.items():
        text = "\n".join(body)
        assert not re.search(r"\bLDG\b", text), f"{n}: LDG in an epilogue-slot kernel"
        assert not re.search(r"\bLD\.", text), f"{n}: generic load in an epilogue-slot kernel"
        assert re.search(r"\bUTMALDG\b", text) and re.search(r"\bUBLKCP\b", text), f"{n}: no TMA / bulk copies"
        assert re.search(r"\bLDS\b", text), f"{n}: the epilogue reads no shared memory"
    # the slot-less instantiations still read their epilogue operands from global memory
    assert any(re.search(r"\bLDG\b", "\n".join(b)) for n, b in funcs.items() if "GemmParamsEpi" not in n)


def test_no_gemm_instantiation_spills():
    out = subprocess.run([_cuobjdump(), "-res-usage", _lib.LIB_PATH], capture_output=True, text=True, check=True).stdout
    lines = out.splitlines()
    usage = {}
    for i, line in enumerate(lines):
        m = re.search(r"Function (\S*gemm_tc_kernel\S*):", line)
        if m and i + 1 < len(lines):
            usage[m.group(1)] = lines[i + 1]
    assert len(usage) >= 10, "no gemm_tc_kernel resource usage found"
    bad = {n: u.strip() for n, u in usage.items() if not re.search(r"\bSTACK:0\b", u) or not re.search(r"\bLOCAL:0\b", u)}
    assert not bad, f"gemm_tc_kernel instantiations with local memory: {bad}"
