"""GPU diagnostics: runs every kernel check (tests/kernel_checks.py and tests/test_attention_tc_gpu.py) in its own
subprocess (a trapping kernel poisons the CUDA context, so isolation keeps the other results); REPORT_JSON = path of a
JSON report."""
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def _checks():
    from tests.kernel_checks import CHECKS
    from tests.test_attention_tc_gpu import CASES      # the attention kernel's pipeline edge cases
    return {**CHECKS, **CASES}


def run_one(name):
    import torch
    r = _checks()[name]()
    torch.cuda.synchronize()
    print("RESULT " + json.dumps(r))


def main():
    names = sys.argv[1:] or sorted(_checks())
    out = {}
    for n in names:
        try:
            p = subprocess.run([sys.executable, __file__, "--one", n], capture_output=True, text=True, timeout=180)
            line = [l for l in p.stdout.splitlines() if l.startswith("RESULT ")]
            if line:
                out[n] = json.loads(line[-1][7:])
            else:
                out[n] = {"ok": False, "rc": p.returncode, "stderr": p.stderr[-1500:], "stdout": p.stdout[-500:]}
        except subprocess.TimeoutExpired:
            out[n] = {"ok": False, "timeout": True}
        print(n, out[n], flush=True)
    if os.environ.get("REPORT_JSON"):            # optional: full JSON report to this path
        with open(os.environ["REPORT_JSON"], "w") as f:
            json.dump(out, f, indent=1)
    bad = [n for n, r in out.items() if not r.get("ok")]
    print(f"{len(out) - len(bad)}/{len(out)} ok; failing: {bad}")


if __name__ == "__main__":
    if len(sys.argv) >= 3 and sys.argv[1] == "--one":
        run_one(sys.argv[2])
    else:
        main()
