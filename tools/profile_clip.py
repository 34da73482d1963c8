"""Per-kernel time of one eager pass of the bench.py headline clip batch (bf16, 264 clips x 10 frames of 32x32 -> 128x128),
taken with torch.profiler (CUDA activities).

  python tools/profile_clip.py --out DIR

DIR/kernels.md and DIR/kernels.json: one row per kernel name with its launches, total device microseconds and share of
the summed kernel time of the pass.  TECO_PROF_CLIPS / TECO_PROF_T / TECO_PROF_LR select another shape."""
import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402
from tecogan_b200 import config, variables as V  # noqa: E402
from tecogan_b200.engine import ClipEngine  # noqa: E402
from tecogan_b200.init_params import xavier_params  # noqa: E402


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--out", required=True, help="output directory")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("profile_clip.py needs a GPU")
    B = int(os.environ.get("TECO_PROF_CLIPS", 264))
    T = int(os.environ.get("TECO_PROF_T", 10))
    LR = int(os.environ.get("TECO_PROF_LR", 32))
    config.set_precision("bf16")
    V.set_default_store(V.VariableStore()).load(xavier_params(1234, 16))
    eng = ClipEngine(LR, LR, T, 16, batch=B, use_graph=False)
    eng.clip_in.copy_(bench.synthetic_clips(T, B, LR, LR, seed=0))
    eng.replay()                      # warm-up: module load, first launches
    torch.cuda.synchronize()
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0.record()
    eng.replay()                      # the same pass without the profiler: the step time the shares are set against
    t1.record()
    torch.cuda.synchronize()
    step_us = t0.elapsed_time(t1) * 1000.0
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        eng.replay()
        torch.cuda.synchronize()
    rows = {}
    for ev in prof.events():
        if ev.device_type == torch.autograd.DeviceType.CUDA and ev.device_time > 0:
            r = rows.setdefault(ev.name, [0, 0.0])
            r[0] += 1
            r[1] += ev.device_time
    total = sum(r[1] for r in rows.values())
    table = sorted(({"kernel": k, "calls": c, "total_us": us, "share": us / total} for k, (c, us) in rows.items()),
                   key=lambda r: -r["total_us"])
    os.makedirs(args.out, exist_ok=True)
    meta = {"clips": B, "frames": T, "lr": LR, "step_us_unprofiled": step_us, "kernel_us_sum": total,
            "gpu": torch.cuda.get_device_name(0)}
    with open(os.path.join(args.out, "kernels.json"), "w") as f:
        json.dump({"meta": meta, "kernels": table}, f, indent=1)
    lines = ["# Kernels of one eager pass: %d clips x %d frames, %dx%d LR, on %s" % (B, T, LR, LR, meta["gpu"]), "",
             "Step %.0f us without the profiler; summed kernel time %.0f us." % (step_us, total), "",
             "| kernel | calls | total us | share |", "|---|---:|---:|---:|"]
    for r in table:
        name = r["kernel"] if len(r["kernel"]) <= 110 else r["kernel"][:107] + "..."
        lines.append("| `%s` | %d | %.0f | %.1f %% |" % (name, r["calls"], r["total_us"], 100.0 * r["share"]))
    with open(os.path.join(args.out, "kernels.md"), "w") as f:
        f.write("\n".join(lines) + "\n")
    print("\n".join(lines[:20]))


if __name__ == "__main__":
    main()
