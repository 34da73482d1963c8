"""The scene cuts of `main.py --scene_threshold` (DESIGN.md section 4.13), measured.

  python tools/bench_scene_cuts.py [--reps 3] [--frames 60] [--out results/bench_scene_cuts.json]

Prints the card's name, power limit and SM clocks (nvidia-smi, in the same call), then:
  * kernel: teco_frame_sad_q8 on one LR frame pair at 540x960 and 1080x1920; CUDA events over 200 launches replayed
    from one CUDA graph after 20 warm-up launches (tools/bench_y4m.py::timed), microseconds per pair against the
    2 * 4 * 3 h w bytes it reads, and that rate's fraction of the H100 SXM's 3.35 TB/s data-sheet HBM3 bandwidth;
  * command: the streaming inference loop on `--frames` seeded 540x960 frames, y4m in -> y4m out (2160x3840),
    num_resblock 16, random weights, bf16.  Three variants alternated `--reps` times: the stream without a cut, without
    and with `--scene_threshold 10` (main.super_resolve_frames / main.super_resolve_scenes), and a stream with a cut
    every 10 frames with the flag.  Wall time from opening the input to the last byte written (the engine is built
    once, before any clock starts, and reset before each run), frames/s, generator steps, the cuts found, and whether
    the two no-cut variants wrote the same bytes.
Temporary files only.
"""
import argparse
import contextlib
import hashlib
import io
import json
import os
import re
import sys
import tempfile
import time

import cv2
import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import bench_y4m as BY  # noqa: E402
from tests import png_cases as PC  # noqa: E402

NRB = 16
LR = (540, 960)
THRESHOLD = 10.0


def bench_kernel():
    from tecogan_b200 import kernels as K
    g = torch.Generator(device="cuda").manual_seed(1)
    res = {}
    for h, w in [(540, 960), (1080, 1920)]:
        a = torch.rand((h, w, 3), device="cuda", generator=g)
        b = torch.rand((h, w, 3), device="cuda", generator=g)
        out = torch.empty(1, dtype=torch.int64, device="cuda")
        res["frame_sad_q8 %dx%d" % (h, w)] = BY.timed(lambda: K.frame_sad_q8(a, b, out), 2 * 4 * 3 * h * w)
    for k, v in res.items():
        print("kernel %s: %s" % (k, json.dumps(v)), flush=True)
    return res


def write_stream(path, n, scene_len, seed):
    """n seeded 540x960 frames as a y4m stream: smooth noise drifting 2 pixels a frame with +-3 grain; a new seed every
    `scene_len` frames (a hard cut), none when scene_len >= n."""
    from tecogan_b200 import y4m
    h, w = LR
    g = np.random.default_rng(seed)
    with open(path, "wb") as f:
        f.write(y4m.format_header(w, h))
        for k in range(n):
            if k % scene_len == 0:
                base = PC.smooth(h, w + 2 * scene_len, seed + k).astype(np.int64)
            j = k % scene_len
            fr = np.clip(base[:, 2 * j:2 * j + w] + g.integers(-3, 4, (h, w, 3)), 0, 255).astype(np.uint8)
            f.write(b"FRAME\n" + cv2.cvtColor(fr, cv2.COLOR_RGB2YUV_I420).tobytes())
    return path


def one_run(eng, src, out, scenes):
    import gc
    import main as M
    from tecogan_b200 import y4m
    eng.reset()
    gc.collect()
    torch.cuda.synchronize()
    log = io.StringIO()
    t0 = time.perf_counter()
    reader = y4m.Y4MReader(src)
    sink = y4m.Y4MWriter(out, 4 * LR[1], 4 * LR[0])
    frames = reader.scenes(THRESHOLD) if scenes else reader.frames()
    try:
        with contextlib.redirect_stdout(log):
            if scenes:
                M.super_resolve_scenes(eng, reader.name, frames, os.path.dirname(out), "output", "jpg", None, sink)
            else:
                M.super_resolve_frames(eng, reader.names(), frames, os.path.dirname(out), "output", "jpg", None, sink)
    finally:
        frames.close()
        sink.close()
    torch.cuda.synchronize()
    wall = time.perf_counter() - t0
    text = log.getvalue()
    with open(out, "rb") as f:
        digest = hashlib.sha256(f.read()).hexdigest()
    os.remove(out)
    steps = int(re.search(r"frame number (\d+)", text).group(1))
    return wall, digest, steps, len(re.findall(r"^scene cut before frame", text, re.M))


def main():
    import main as M
    from tecogan_b200 import config, variables as V
    from tecogan_b200.engine import InferenceEngine
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--frames", type=int, default=60)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_scene_cuts: needs a CUDA device")
    res = {"card": BY.card()}
    print("card:", res["card"], flush=True)
    res["kernel"] = bench_kernel()
    config.set_precision("bf16")
    M.load_checkpoint(V.set_default_store(V.VariableStore(seed=1)), "random:5", NRB)
    variants = {"no_cut_plain": ("plain", False), "no_cut_flag": ("plain", True), "cut_every_10_flag": ("cuts", True)}
    with tempfile.TemporaryDirectory() as tmp:
        eng = InferenceEngine(LR[0], LR[1], NRB)
        warm = write_stream(os.path.join(tmp, "warm.y4m"), 12, 6, seed=3)
        for name, (_, scenes) in variants.items():          # module loads, graph captures, allocator
            one_run(eng, warm, os.path.join(tmp, "warm_out.y4m"), scenes)
        streams = {"plain": write_stream(os.path.join(tmp, "plain.y4m"), a.frames, a.frames, seed=7),
                   "cuts": write_stream(os.path.join(tmp, "cuts.y4m"), a.frames, 10, seed=7)}
        runs, digests = {v: [] for v in variants}, {}
        for rep in range(a.reps):
            for name, (stream, scenes) in variants.items():
                wall, digest, steps, cuts = one_run(eng, streams[stream], os.path.join(tmp, "out.y4m"), scenes)
                digests.setdefault(name, set()).add(digest)
                runs[name].append({"wall_s": round(wall, 3), "fps": round(a.frames / wall, 2), "steps": steps,
                                   "cuts": cuts, "sm_clock_after": BY.sm_clock()})
                print("%s rep %d: %s" % (name, rep, json.dumps(runs[name][-1])), flush=True)
        med = {k: float(np.median([r["wall_s"] for r in v])) for k, v in runs.items()}
        res["command"] = {
            "frames": "%d x %dx%d -> %dx%d, y4m -> y4m" % (a.frames, LR[0], LR[1], 4 * LR[0], 4 * LR[1]),
            "threshold": THRESHOLD, "runs": runs, "median_wall_s": med,
            "flag_overhead_no_cut": round(med["no_cut_flag"] / med["no_cut_plain"] - 1, 4),
            "no_cut_outputs_identical": len(digests["no_cut_plain"] | digests["no_cut_flag"]) == 1,
            "each_variant_repeatable": all(len(v) == 1 for v in digests.values())}
        print("command: %s" % json.dumps(res["command"]), flush=True)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
