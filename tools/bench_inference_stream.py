"""The streaming inference command (main.super_resolve_frames over lib/dataloader.py::stream_inputs: decode a window
ahead on a reader thread, encode and write behind on a writer thread) against the serial loop it replaced, restated
below: every input decoded and resident first, then per frame one step, a device synchronise and save_img.

  python tools/bench_inference_stream.py [--reps 3] [--out results/bench_inference_stream.json]

Prints the card's name and power limit, then for seeded PNG sequences written by cv2.imwrite (smooth moving frames with
noise) -- 41 x 144x180 (Vid4 size), 300 x 270x480 (1080p output), 120 x 540x960 (4K output) -- and for PNG and JPEG
output, old and new alternated `--reps` times each (num_resblock 16, random weights, bf16): the loop's wall time from
the file list to the last file written (the engine is built before the clock starts and captures its graphs inside
it, for both), frames/s, peak device memory above what was allocated before the loop, and whether every run wrote the
same files as the first serial run.  Temporary files only.
"""
import argparse
import contextlib
import hashlib
import io
import json
import os
import shutil
import subprocess
import sys
import tempfile
import time

import cv2
import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tests import png_cases as PC  # noqa: E402

SEQS = [(144, 180, 41), (270, 480, 300), (540, 960, 120)]
EXTS = ["png", "jpg"]
NRB = 16


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip()


def write_frames(d, h, w, n, seed):
    os.makedirs(d, exist_ok=True)
    g = np.random.default_rng(seed)
    base = PC.smooth(h, w + 2 * n, seed).astype(np.int64)
    for k in range(n):
        f = np.clip(base[:, 2 * k:2 * k + w] + g.integers(-3, 4, (h, w, 3)), 0, 255).astype(np.uint8)
        cv2.imwrite(os.path.join(d, "%04d.png" % (k + 1)), np.ascontiguousarray(f[:, :, ::-1]))
    return d


def serial_loop(eng, paths, image_dir, ext):
    """The parent's command: read_inputs of the whole sequence, then per frame step, synchronise, save_img."""
    from tecogan_b200.lib.dataloader import padded, read_inputs
    from tecogan_b200.lib.ops import save_img
    inputs = padded(read_inputs(paths, False))
    names = padded(paths)
    for i in range(len(inputs)):
        out = eng.step(inputs[i], next_lr=inputs[i + 1] if i + 1 < len(inputs) else None)
        torch.cuda.synchronize()
        if i >= 5:
            stem = os.path.splitext(os.path.basename(names[i]))[0]
            save_img(os.path.join(image_dir, "output_%s.%s" % (stem, ext)), out[0])


def stream_loop(eng, paths, image_dir, ext):
    import main as M
    from tecogan_b200.lib.dataloader import padded, stream_inputs
    frames = stream_inputs(paths, False)
    try:
        M.super_resolve_frames(eng, padded(paths), frames, image_dir, "output", ext)
    finally:
        frames.close()


def digest(d):
    h = hashlib.sha256()
    for n in sorted(os.listdir(d)):
        h.update(n.encode())
        with open(os.path.join(d, n), "rb") as f:
            h.update(f.read())
    return h.hexdigest()


def one_run(loop, paths, h, w, out_dir):
    import gc
    from tecogan_b200.engine import InferenceEngine
    os.makedirs(out_dir)
    eng = InferenceEngine(h, w, NRB)
    gc.collect()
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    t0 = time.perf_counter()
    with contextlib.redirect_stdout(io.StringIO()):
        loop(eng, paths, out_dir, out_dir.rsplit(".", 1)[-1])
    torch.cuda.synchronize()
    wall = time.perf_counter() - t0
    peak = torch.cuda.max_memory_allocated() - base
    del eng
    files = digest(out_dir)
    shutil.rmtree(out_dir)
    return wall, peak, files


def main():
    import main as M
    from tecogan_b200 import config, variables as V
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_inference_stream: needs a CUDA device")
    res = {"card": card(), "runs": {}}
    print("card:", res["card"], flush=True)
    config.set_precision("bf16")
    M.load_checkpoint(V.set_default_store(V.VariableStore(seed=1)), "random:5", NRB)
    with tempfile.TemporaryDirectory() as tmp:
        for h, w, n in SEQS:
            d = write_frames(os.path.join(tmp, "seq_%dx%d" % (h, w)), h, w, n, seed=h + w)
            paths = sorted(os.path.join(d, f) for f in os.listdir(d))
            if (h, w, n) == SEQS[0]:               # warm-up, not recorded: module loads, encoder plans, allocator
                for ext in EXTS:
                    for kind, loop in (("serial", serial_loop), ("stream", stream_loop)):
                        one_run(loop, paths, h, w, os.path.join(tmp, "warm_%s.%s" % (kind, ext)))
            for ext in EXTS:
                key = "%d x %dx%d -> %dx%d %s" % (n, h, w, 4 * h, 4 * w, ext)
                r = {"serial": [], "stream": []}
                ref = None
                for rep in range(a.reps):
                    for kind, loop in (("serial", serial_loop), ("stream", stream_loop)):
                        wall, peak, files = one_run(loop, paths, h, w, os.path.join(tmp, "out_%s_%d.%s" % (kind, rep, ext)))
                        ref = files if ref is None else ref
                        r[kind].append({"wall_s": wall, "fps": n / wall, "peak_MiB": peak / 2 ** 20, "identical": files == ref})
                res["runs"][key] = r
                line = {k: {"wall_s": [round(x["wall_s"], 3) for x in v], "fps": [round(x["fps"], 1) for x in v],
                            "peak_MiB": [round(x["peak_MiB"], 1) for x in v], "identical": all(x["identical"] for x in v)}
                        for k, v in r.items()}
                print("%s: %s" % (key, json.dumps(line)), flush=True)
            shutil.rmtree(d)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
