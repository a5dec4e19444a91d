"""Evidence run for the attention controllers (SURVEY.md 8f-2) (REPORT_JSON = path of a JSON report):
explicit-probability attention vs torch, the hook vs the oracle's hook, the device-native controllers replayed against the
fixtures the reference's own classes produced, the whole `use_blend: true` flow vs the oracle, and what controller mode costs
per step at the benchmark size (eager, host callback per controlled layer) next to the CUDA-graph step."""
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    import torch
    from tests import p2p_checks as P
    from tests import unet_checks as U
    from videoswap_b200 import DDIMScheduler, VideoSwapPipeline, p2p
    out = {}
    out["explicit_attention_d160_n256"] = P.explicit_attention_check(B=3, N=256, C=1280)
    out["explicit_cross_attention_d160"] = P.explicit_attention_check(B=4, N=256, NK=77, C=1280, kv_div=2, seed=172)
    out["hook_vs_oracle_32x32_latent"] = {k: v for k, v in P.unet_hook_vs_oracle(Fr=2, hw=32).items() if k != "order"}
    out["hook_with_edit_vs_oracle"] = {k: v for k, v in P.unet_hook_vs_oracle(Fr=2, hw=16, edit=True).items() if k != "order"}
    for kind in ("refine", "replace"):
        out[f"controllers_vs_reference_fixture_{kind}"] = P.replay_vs_reference_fixture(kind)
    t0 = time.time()
    out["use_blend_flow_2+2_steps_64x64"] = P.edit_flow_vs_oracle(n_steps=2)
    out["use_blend_flow_seconds"] = time.time() - t0
    # ---- cost of controller mode at the benchmark size: one CFG step, 16 frames 64x64, store controller registered
    m, _ = U.get_model()
    pipe = VideoSwapPipeline(m, DDIMScheduler())
    pipe.scheduler.set_timesteps(50)
    lat = U.randn((1, 4, 16, 64, 64), 5).half().cuda()
    emb = U.randn((2, 16, 77, 768), 6).half().cuda()
    store = p2p.AttentionStore(keep_all_steps=False)
    p2p.register_attention_control(pipe, store)
    try:
        for _ in range(2):
            x = pipe.step(lat, 981, emb, 7.5)
            store.step_callback(x)
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(3):
            x = pipe.step(lat, 981, emb, 7.5)
            store.step_callback(x)
        e1.record()
        torch.cuda.synchronize()
        out["controller_mode_ms_per_step_c2"] = e0.elapsed_time(e1) / 3
        out["stored_bytes_per_step"] = sum(t.numel() * t.element_size() for v in store.attention_store.values() for t in v) // 2
    finally:
        p2p.register_attention_control(pipe, None)
    if os.environ.get("REPORT_JSON"):            # optional: full JSON report to this path
        with open(os.environ["REPORT_JSON"], "w") as f:
            json.dump(out, f, indent=1)
    print(json.dumps(out)[:3000])


if __name__ == "__main__":
    main()
