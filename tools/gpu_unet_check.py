"""GPU diagnostics: whole-UNet parity with per-stage taps (REPORT_JSON = path of a JSON report)."""
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    import torch
    from tests import unet_checks as U
    out = {}
    t0 = time.time()
    for name, fn in [("golden", U.unet_vs_reference_golden),
                     ("oracle_small_taps", lambda: U.unet_vs_oracle(B=1, Fr=2, hw=8, edlora=True, taps=True)),
                     ("oracle_cfg_res", lambda: U.unet_vs_oracle(B=2, Fr=3, hw=16, edlora=True, residuals=True, taps=True)),
                     ("pipeline3", lambda: U.pipeline_vs_oracle(steps=3)),
                     ("adapter", U.adapter_vs_golden)]:
        try:
            out[name] = fn()
        except Exception as e:  # noqa: BLE001
            import traceback
            out[name] = {"error": repr(e), "tb": traceback.format_exc()[-2000:]}
        print(name, json.dumps(out[name])[:3000], time.time() - t0, flush=True)
    if os.environ.get("REPORT_JSON"):            # optional: full JSON report to this path
        with open(os.environ["REPORT_JSON"], "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
