"""CPU test on the compiled sm_90a code of the built library (no GPU needed).

ptxas serialises every wgmma of a function that contains a CALL (warning C7510, "wgmma pipeline crossing function
boundary"): each HGMMA then waits for its own completion and the asynchronous main loops lose their overlap.  A
`printf` in device code is such a call, so no kernel that issues wgmma may contain one.
"""
import os
import re
import shutil
import subprocess

from videoswap_b200 import _lib


def _cuobjdump() -> str:
    for cand in (shutil.which("cuobjdump"), "/usr/local/cuda/bin/cuobjdump"):
        if cand and os.path.exists(cand):
            return cand
    nvcc = shutil.which("nvcc")
    assert nvcc, "neither cuobjdump nor nvcc found"
    return os.path.join(os.path.dirname(nvcc), "cuobjdump")


def _sass_functions(lib_path: str) -> dict:
    out = subprocess.run([_cuobjdump(), "-sass", lib_path], capture_output=True, text=True, check=True).stdout
    funcs, name = {}, None
    for line in out.splitlines():
        m = re.match(r"\s*Function : (\S+)", line)
        if m:
            name = m.group(1)
            funcs[name] = []
        elif name is not None:
            funcs[name].append(line)
    return funcs


def _leaves_function(body) -> bool:
    """A CALL out of the function: by register (CALL.ABS, e.g. vprintf) or to an address past its end.  ptxas's own
    out-of-line slow paths (e.g. of an IEEE division) are CALL.REL to a subroutine inside the function's code; they do
    not serialise wgmma."""
    addrs = [int(m.group(1), 16) for l in body if (m := re.match(r"\s*/\*([0-9a-f]{4,})\*/", l))]
    end = max(addrs, default=0)
    for l in body:
        m = re.search(r"\bCALL(\.\S+)?\s+(\S+)", l)
        if m is None:
            continue
        target = m.group(2).rstrip(";")
        if not target.startswith("0x") or int(target, 16) > end:
            return True
    return False


def test_no_call_in_any_wgmma_kernel():
    funcs = _sass_functions(_lib.LIB_PATH)
    wgmma = {n: body for n, body in funcs.items() if any("HGMMA" in l for l in body)}
    assert any("gemm_tc_kernel" in n for n in wgmma), "no wgmma GEMM kernel found in the library"
    assert any("attn_tc_kernel" in n for n in wgmma), "no wgmma attention kernel found in the library"
    bad = sorted(n for n, body in wgmma.items() if _leaves_function(body))
    assert not bad, f"{len(bad)} wgmma kernels contain a CALL (wgmma serialised): {bad[:3]}"
