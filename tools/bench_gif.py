"""Cost of the GIF training summaries (Network.image_summary, tecogan_b200.gif).

  python tools/bench_gif.py [--reps 20] [--steps 20] [--out results/bench_gif.json]

Prints the card's name, power limit and max SM clock, then:
  * the device time of one summary -- the four quantisations and the 16 encodes (min(4, B) clips of LR, HR, Generated
    and WarpPreGen) -- at the default configuration (B = 4, crop 32, RNN_N 10: LR 4x10x32^2, HR and Generated
    4x10x128^2, WarpPreGen 4x9x128^2) and with --pingpang (19 and 18 frames): CUDA events around the launches, warmed,
    median of --reps; and the wall time of the same with the copies back to the host;
  * a per-kernel split of one summary from a separate torch.profiler run;
  * cv2.imencodeanimation('.gif') of the same 16 animations on this host's CPU, as context only: its own quantiser
    writes different bytes;
  * the bf16 TecoGAN training step (config of record: 16 residual blocks, ping-pong, VGG 0.2) over the same --steps
    steps without and with Network.image_summary after every step, alternating in blocks of 5.
Seeded smooth frames stand in for the tensors; the summary's cost does not depend on the weights.
"""
import argparse
import json
import os
import re
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip()


def tensors(B, T, crop, seed=0):
    """fp32 stand-ins: LR [B,T,crop,crop,3] in [0,1], HR / Generated [B,T,4crop,4crop,3] and WarpPreGen [B,T-1,...] in
    [-1,1], smooth with a little noise (content like a training clip's)."""
    g = torch.Generator(device="cuda").manual_seed(seed)

    def clip(t, s, lo):
        y = torch.linspace(0, 3, s, device="cuda").view(1, 1, s, 1, 1)
        x = torch.linspace(0, 3, s, device="cuda").view(1, 1, 1, s, 1)
        k = torch.arange(t, device="cuda", dtype=torch.float32).view(1, t, 1, 1, 1)
        ph = torch.rand((B, 1, 1, 1, 3), generator=g, device="cuda") * 6
        v = 0.5 + 0.45 * torch.sin(x + 2 * y + 0.3 * k + ph) + 0.02 * torch.randn((B, t, s, s, 3), generator=g, device="cuda")
        v = v.clamp(0, 1)
        return (v if lo == 0 else v * 2 - 1).contiguous()
    return {"LR": clip(T, crop, 0), "HR": clip(T, 4 * crop, -1), "Generated": clip(T, 4 * crop, -1),
            "WarpPreGen": clip(T - 1, 4 * crop, -1)}


def summary_launch(src, enc):
    from tecogan_b200.gif import convert_image_u8
    k = min(4, src["LR"].shape[0])
    return [enc[n].launch(convert_image_u8(x[:k], deprocess=(n != "LR"))) for n, x in src.items()]


def time_summary(src, reps):
    from tecogan_b200._encode import collect
    from tecogan_b200.gif import GifEncoder
    enc = {n: GifEncoder(n) for n in src}
    for _ in range(3):
        collect(summary_launch(src, enc))
    dev, wall = [], []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        a.record()
        pending = summary_launch(src, enc)
        b.record()
        files = collect(pending)
        wall.append((time.perf_counter() - t0) * 1e3)
        dev.append(a.elapsed_time(b))
    nbytes = sum(len(f) for fs in files for f in fs)
    prof = {}
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as p:
        collect(summary_launch(src, enc))
        torch.cuda.synchronize()
    for e in p.key_averages():
        m = re.search(r"(gif_\w+|convert_image_u8_kernel)", e.key)
        if m and e.device_time_total > 0:
            prof[m.group(1)] = round(prof.get(m.group(1), 0.0) + e.device_time_total / 1e3, 3)
    return {"device_ms_median": float(np.median(dev)), "device_ms_min": float(np.min(dev)),
            "wall_ms_median": float(np.median(wall)), "bytes": nbytes, "kernels_ms": prof}


def time_cv2(src, reps=3):
    import cv2
    from tecogan_b200.gif import convert_image_u8
    k = min(4, src["LR"].shape[0])
    anims = []
    for n, x in src.items():
        u8 = convert_image_u8(x[:k], deprocess=(n != "LR")).cpu().numpy()
        for i in range(k):
            a = cv2.Animation()
            a.frames = [np.ascontiguousarray(f[:, :, ::-1]) for f in u8[i]]
            a.durations = [330] * len(u8[i])
            a.loop_count = 0
            anims.append(a)
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        for a in anims:
            ok, _ = cv2.imencodeanimation(".gif", a)
            assert ok
        ts.append((time.perf_counter() - t0) * 1e3)
    return {"host_ms_median": float(np.median(ts)), "cpus": os.cpu_count()}


def time_training(steps):
    import main as M
    from tecogan_b200 import config, variables as V
    from tecogan_b200.init_params import xavier_params
    from tecogan_b200.lib.dataloader import frvsr_gpu_data_loader
    from tecogan_b200.lib.Teco import TecoGAN
    F = M.parse_flags(["--mode", "train", "--output_dir", "/tmp/x", "--num_resblock", "16", "--ratio", "0.01",
                       "--pingpang", "--pp_scaling", "0.5", "--vgg_scaling", "0.2", "--learning_rate", "0.00005",
                       "--decay_rate", "1.0", "--stair", "--train_precision", "bf16"])
    config.set_train_precision("bf16")
    V.set_default_store(V.VariableStore()).load(xavier_params(1, F.num_resblock, True, True))
    dev = torch.device("cuda")
    lr, tg = frvsr_gpu_data_loader(M.synthetic_hr_batch(F, 0, 0, dev), F)
    Net = TecoGAN(lr, tg, F)
    for _ in range(3):
        Net.train(lr, tg)
        Net.image_summary()
    torch.cuda.synchronize()
    plain, with_s = [], []
    for blk in range(2 * ((steps + 4) // 5)):
        summ = blk % 2 == 1
        for _ in range(5):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            Net.train(lr, tg)
            if summ:
                Net.image_summary()
            torch.cuda.synchronize()
            (with_s if summ else plain).append((time.perf_counter() - t0) * 1e3)
    return {"step_ms_median": float(np.median(plain)), "step_plus_summary_ms_median": float(np.median(with_s)),
            "steps_each": len(plain)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "bench_gif needs a GPU"
    res = {"card": card()}
    print("card:", res["card"])
    for name, T in (("default", 10), ("pingpang", 19)):
        src = tensors(4, T, 32)
        r = time_summary(src, a.reps)
        r["cv2_imencodeanimation"] = time_cv2(src)
        res[name] = r
        print(name, json.dumps(r))
    res["training_bf16_tecogan"] = time_training(a.steps)
    print("training", json.dumps(res["training_bf16_tecogan"]))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
