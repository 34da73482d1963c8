"""The output resize of `main.py --outscale` (DESIGN.md section 4.11), measured two ways.

  python tools/bench_outscale.py [--reps 3] [--frames 60] [--out results/bench_outscale.json]

Prints the card's name, power limit and SM clocks (nvidia-smi, in the same call), then:
  * kernel: teco_resize_lanczos4_u8 alone, CUDA events over 100 launches after 10 warm-up launches, microseconds per
    frame for 4320x7680 -> 2160x3840, 2160x3840 -> 1620x2880 and 1080x1920 -> 2160x3840, with the bytes the kernel
    must move (source frame read once, output written once, from the shapes) and that rate's fraction of the H100 SXM's
    3.35 TB/s data-sheet HBM3 bandwidth;
  * command: the streaming inference loop (main.super_resolve_frames over stream_inputs) on `--frames` seeded
    1080x1920 PNG frames, num_resblock 16, random weights, bf16, JPEG output, in three variants alternated `--reps`
    times: `--outscale 2` (4K files, resized on the device), no flag (8K files) and `--outscale 2` with the resize
    done on the host by cv2.resize on the writer thread (restated below, not part of the package: the frame is copied
    back at 8K, resized and written by cv2.imwrite).  Wall time from the file list to the last file written (the engine
    is built once, before any clock starts, and reset before each run), frames/s, whether each variant wrote the same
    bytes in every run and whether both 4K variants wrote the same bytes.
Temporary files only.
"""
import argparse
import contextlib
import hashlib
import io
import json
import os
import queue
import shutil
import subprocess
import sys
import tempfile
import threading
import time

import cv2
import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tests import png_cases as PC  # noqa: E402

KERNEL_CASES = [((4320, 7680), (2160, 3840)), ((2160, 3840), (1620, 2880)), ((1080, 1920), (2160, 3840))]
HBM_BYTES_PER_S = 3.35e12           # H100 SXM data sheet, HBM3
NRB = 16
LR = (1080, 1920)
SCALE = 2.0


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip()


def sm_clock():
    """The SM clock now, read right after a timed loop (an idle card reports its idle clock)."""
    q = subprocess.run(["nvidia-smi", "--query-gpu=clocks.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip()


def bench_kernel(src_hw, dst_hw, warm=10, iters=100):
    from tecogan_b200 import kernels as K
    from tecogan_b200 import resize as RZ
    g = torch.Generator(device="cuda").manual_seed(src_hw[1])
    src = torch.randint(0, 256, src_hw + (3,), dtype=torch.uint8, device="cuda", generator=g)
    dst = torch.empty(dst_hw + (3,), dtype=torch.uint8, device="cuda")
    tabs = RZ.tables(*src_hw, *dst_hw, src.device)
    for _ in range(warm):
        K.resize_lanczos4(src, dst, tabs)
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0.record()
    for _ in range(iters):
        K.resize_lanczos4(src, dst, tabs)
    t1.record()
    torch.cuda.synchronize()
    us = t0.elapsed_time(t1) * 1e3 / iters
    moved = src.numel() + dst.numel()
    return {"us_per_frame": round(us, 2), "bytes": moved, "GB_per_s": round(moved / us / 1e3, 1),
            "fraction_of_3.35TB_per_s": round(moved / (us * 1e-6) / HBM_BYTES_PER_S, 3)}


class HostResizeWriter:
    """FrameWriter's interface with the resize on the host: put() copies the 4x frame back to a pinned buffer on the
    producer's stream; the writer thread waits for it, runs cv2.resize(INTER_LANCZOS4) and cv2.imwrite."""

    def __init__(self, h, w, device):
        self.h, self.w, self.error = h, w, None
        self.jobs, self.free, self.made = queue.Queue(), queue.Queue(), 0
        self.thread = threading.Thread(target=self._run, daemon=True)
        self.thread.start()

    def put(self, out_u8, path):
        if self.made < 3 and self.free.empty():
            self.made += 1
            self.free.put((torch.empty(out_u8.shape, dtype=torch.uint8, pin_memory=True), torch.cuda.Event()))
        slot = self.free.get()
        if isinstance(slot, BaseException):
            raise slot
        slot[0].copy_(out_u8, non_blocking=True)
        slot[1].record()
        self.jobs.put((path, slot))

    def _run(self):
        try:
            while True:
                item = self.jobs.get()
                if item is None:
                    return
                path, (host, ev) = item
                ev.synchronize()
                small = cv2.resize(host.numpy(), (self.w, self.h), interpolation=cv2.INTER_LANCZOS4)
                cv2.imwrite(path, np.ascontiguousarray(small[:, :, ::-1]))
                self.free.put((host, ev))
        except BaseException as e:
            self.error = e
            self.free.put(e)

    def close(self):
        self.jobs.put(None)
        self.thread.join()


def write_frames(d, h, w, n, seed):
    os.makedirs(d, exist_ok=True)
    g = np.random.default_rng(seed)
    base = PC.smooth(h, w + 2 * n, seed).astype(np.int64)
    for k in range(n):
        f = np.clip(base[:, 2 * k:2 * k + w] + g.integers(-3, 4, (h, w, 3)), 0, 255).astype(np.uint8)
        cv2.imwrite(os.path.join(d, "%04d.png" % (k + 1)), np.ascontiguousarray(f[:, :, ::-1]))
    return d


def digest(d):
    h = hashlib.sha256()
    for n in sorted(os.listdir(d)):
        h.update(n.encode())
        with open(os.path.join(d, n), "rb") as f:
            h.update(f.read())
    return h.hexdigest()


def one_run(eng, paths, out_dir, out_hw, host_resize):
    import gc
    import main as M
    from tecogan_b200.lib import writer as W
    from tecogan_b200.lib.dataloader import padded, stream_inputs
    os.makedirs(out_dir)
    eng.reset()                                   # every run starts the recurrence afresh, as a new command does
    gc.collect()
    torch.cuda.synchronize()
    real = W.FrameWriter
    if host_resize:
        W.FrameWriter = HostResizeWriter
    t0 = time.perf_counter()
    try:
        frames = stream_inputs(paths, False)
        try:
            with contextlib.redirect_stdout(io.StringIO()):
                M.super_resolve_frames(eng, padded(paths), frames, out_dir, "output", "jpg", out_hw)
        finally:
            frames.close()
        torch.cuda.synchronize()
    finally:
        W.FrameWriter = real
    wall = time.perf_counter() - t0
    files = digest(out_dir)
    shutil.rmtree(out_dir)
    return wall, files


def main():
    import main as M
    from tecogan_b200 import config, resize as RZ, variables as V
    from tecogan_b200.engine import InferenceEngine
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--frames", type=int, default=60)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_outscale: needs a CUDA device")
    res = {"card": card(), "cv2_threads": cv2.getNumThreads(), "kernel": {}, "command": {}}
    print("card:", res["card"], "| cv2 threads:", res["cv2_threads"], flush=True)
    for src_hw, dst_hw in KERNEL_CASES:
        key = "%dx%d -> %dx%d" % (src_hw + dst_hw)
        res["kernel"][key] = bench_kernel(src_hw, dst_hw)
        res["kernel"][key]["sm_clock_after"] = sm_clock()
        print("kernel %s: %s" % (key, json.dumps(res["kernel"][key])), flush=True)
    config.set_precision("bf16")
    M.load_checkpoint(V.set_default_store(V.VariableStore(seed=1)), "random:5", NRB)
    out_hw = RZ.out_size(LR[0], LR[1], SCALE)
    variants = [("outscale_device", out_hw, False), ("no_flag_8k", None, False), ("outscale_cv2_host", out_hw, True)]
    with tempfile.TemporaryDirectory() as tmp:
        d = write_frames(os.path.join(tmp, "seq"), LR[0], LR[1], a.frames, seed=7)
        paths = sorted(os.path.join(d, f) for f in os.listdir(d))
        eng = InferenceEngine(LR[0], LR[1], NRB)
        warm = paths[:8]                          # module loads, encoder plans, tables, allocator
        for name, hw, host in variants:
            one_run(eng, warm, os.path.join(tmp, "warm_" + name), hw, host)
        runs = {name: [] for name, _, _ in variants}
        digests = {}
        for rep in range(a.reps):
            for name, hw, host in variants:
                wall, files = one_run(eng, paths, os.path.join(tmp, "out_%s_%d" % (name, rep)), hw, host)
                digests.setdefault(name, set()).add(files)
                runs[name].append({"wall_s": round(wall, 3), "fps": round(a.frames / wall, 2), "sm_clock_after": sm_clock()})
                print("%s rep %d: %s" % (name, rep, json.dumps(runs[name][-1])), flush=True)
        res["command"] = {
            "frames": "%d x %dx%d -> %dx%d jpg (--outscale %g); no flag %dx%d" % (
                a.frames, LR[0], LR[1], out_hw[0], out_hw[1], SCALE, 4 * LR[0], 4 * LR[1]),
            "runs": runs,
            "4k_files_identical": len(digests["outscale_device"] | digests["outscale_cv2_host"]) == 1,
            "each_variant_repeatable": all(len(v) == 1 for v in digests.values())}
        print("command: %s" % json.dumps(res["command"]), flush=True)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
