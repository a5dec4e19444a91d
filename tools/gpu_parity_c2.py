"""Parity at the BENCHMARKED configuration (VERDICT r1, item 1): one full CFG denoise step on latents [1,4,16,64,64]
(UNet batch 2, ED-LoRA embeddings [2,16,77,768], adapter residuals) through the native path -- eager AND the CUDA-graph
replay bench.py times -- against the CPU fp32 oracle, with per-block taps.  ~3 min of CPU time.
With REPORT_JSON set, writes the full report (per-block taps) there."""
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    import torch
    from oracle import unet3d_oracle as O
    from tests import unet_checks as U
    from videoswap_b200 import DDIMScheduler, VideoSwapPipeline, ops
    from videoswap_b200.pipeline import GraphedStep
    torch.set_num_threads(min(os.cpu_count() or 1, 32))
    Fr = int(os.environ.get("C2_FRAMES", 16))
    hw = 64
    t0 = time.time()
    m, sd = U.get_model()
    boc = m.cfg.block_out_channels
    lat = U.randn((1, 4, Fr, hw, hw), 71).half()
    ehs2 = U.randn((2, 16, 77, 768), 72).half()                      # uncond first
    res = [(0.5 * U.randn((Fr, c, hw >> l, hw >> l), 80 + l)).half() for l, c in enumerate(boc)]   # adapter maps, per frame
    res2 = [torch.cat([r, r]) for r in res]                          # duplicated for CFG (pipeline_videoswap.py:548-550)
    t, guidance = 981, 7.5
    out = {"config": f"latents [1,4,{Fr},{hw},{hw}] fp16, CFG {guidance} (UNet batch 2), ED-LoRA embeds [2,16,77,768], adapter residuals, t={t}"}

    # ---- native: UNet forward with taps, then the step (eager) and the captured graph
    ntaps = {}
    x2 = torch.cat([lat, lat]).cuda()
    eps = m(x2, t, ehs2.cuda(), down_block_additional_residuals=[r.cuda() for r in res2], return_dict=False, _taps=ntaps)[0]
    torch.cuda.synchronize()
    ntaps = {k: v.cpu() for k, v in ntaps.items()}
    pipe = VideoSwapPipeline(m, DDIMScheduler())
    pipe.scheduler.set_timesteps(50)
    nat_step = pipe.step(lat.cuda(), t, ehs2.cuda(), guidance, [r.cuda() for r in res2])
    g = GraphedStep(pipe, lat.cuda(), ehs2.cuda(), guidance, [r.cuda() for r in res2])
    nat_graph = g(lat.cuda(), t).clone()
    nat_graph2 = g(lat.cuda(), t).clone()
    torch.cuda.synchronize()
    out["native_s"] = time.time() - t0
    out["graph_vs_eager_psnr"] = U.psnr(nat_graph, nat_step.float().cpu())
    out["graph_replay_bit_identical"] = bool(torch.equal(nat_graph, nat_graph2))

    # ---- oracle: the two CFG halves are independent through the UNet (GroupNorm statistics are per batch element), so
    #      they run one after the other to bound the host memory of the materialised N = 4096 score matrices
    t1 = time.time()
    otaps = [{}, {}]
    halves = []
    with torch.no_grad():
        for b in range(2):
            halves.append(O.unet_forward(sd, O.OracleConfig(), lat.float(), t, ehs2[b:b + 1].float(), [r.float() for r in res],
                                         taps=otaps[b]))
        ref_eps = torch.cat(halves)
        sched = O.DDIM()
        ref_step = sched.step(O.cfg_combine(ref_eps, guidance), t, lat.float(), 50)
    out["oracle_s"] = time.time() - t1
    out["eps"] = {"psnr": U.psnr(eps, ref_eps), "max_err": (eps.float().cpu() - ref_eps).abs().max().item(),
                  "ref_max": ref_eps.abs().max().item(), "finite": bool(torch.isfinite(eps).all().item())}
    out["step_eager"] = {"psnr": U.psnr(nat_step, ref_step), "max_err": (nat_step.float().cpu() - ref_step).abs().max().item()}
    out["step_graph"] = {"psnr": U.psnr(nat_graph, ref_step), "max_err": (nat_graph.float().cpu() - ref_step).abs().max().item()}
    taps = {}
    for k, v in ntaps.items():
        if k in otaps[0]:
            ref = torch.cat([otaps[0][k], otaps[1][k]])
            o = U.nhwc_tap_to_ncfhw(v, 2)
            taps[k] = {"psnr": U.psnr(o, ref), "max_err": (o - ref).abs().max().item(), "ref_max": ref.abs().max().item()}
    out["taps"] = taps
    out["min_tap_psnr"] = min(v["psnr"] for v in taps.values()) if taps else None
    out["ok"] = bool(out["eps"]["finite"] and out["eps"]["psnr"] >= 40 and out["step_graph"]["psnr"] >= 40 and
                     (out["min_tap_psnr"] is None or out["min_tap_psnr"] >= 40))
    if os.environ.get("REPORT_JSON"):            # optional: full JSON report to this path
        with open(os.environ["REPORT_JSON"], "w") as f:
            json.dump(out, f, indent=1)
    print(json.dumps({k: v for k, v in out.items() if k != "taps"}))
    sys.exit(0 if out["ok"] else 1)


if __name__ == "__main__":
    main()
