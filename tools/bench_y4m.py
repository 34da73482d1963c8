"""The YUV4MPEG2 input and output of `main.py --input_y4m / --output_y4m` (DESIGN.md section 4.12), measured two ways.

  python tools/bench_y4m.py [--reps 3] [--frames 60] [--out results/bench_y4m.json]

Prints the card's name, power limit and SM clocks (nvidia-smi, in the same call), then:
  * kernels: teco_rgb_to_i420_u8 at 2160x3840 and 4320x7680 and teco_i420_to_rgb_u8 at 540x960 and 1080x1920 (one
    frame per launch), alone and -- for the input side -- followed by the frames_to_f32 launch the reader makes; CUDA
    events over 200 launches after 20 warm-up launches (a kernel alone replayed from one CUDA graph, so that Python's
    launch rate does not bound it; the reader's pair launched from Python, as the reader launches it), microseconds per
    frame, the bytes the kernel must move (its
    input read once and its output written once, from the shapes) and that rate's fraction of the H100 SXM's 3.35 TB/s
    data-sheet HBM3 bandwidth;
  * command: the streaming inference loop (main.super_resolve_frames) on `--frames` seeded 540x960 frames, 2160x3840
    out, num_resblock 16, random weights, bf16, in three variants alternated `--reps` times: y4m in -> y4m out, PNG
    files in -> JPEG files out (the default path), and y4m in -> y4m out with the RGB -> I420 conversion done on the
    host by cv2.cvtColor on the writer thread (restated below, not part of the package: each 4K RGB frame is copied
    back, converted and written).  Wall time from opening the input to the last byte written (the engine is built
    once, before any clock starts, and reset before each run), frames/s, whether each variant wrote the same bytes in
    every run and whether both y4m variants wrote the same bytes.
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

HBM_BYTES_PER_S = 3.35e12           # H100 SXM data sheet, HBM3
NRB = 16
LR = (540, 960)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip()


def sm_clock():
    """The SM clock now, read right after a timed loop (an idle card reports its idle clock)."""
    q = subprocess.run(["nvidia-smi", "--query-gpu=clocks.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip()


def timed(fn, moved, warm=20, iters=200, graph=True):
    """Microseconds per call of fn over `iters` calls after `warm`.  graph=True captures the iters launches in one CUDA
    graph and times its replay, so the number is the kernels' and not Python's launch rate; graph=False times the calls
    as the program makes them."""
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    if graph:
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            for _ in range(iters):
                fn()
        g.replay()
        run = g.replay
    else:
        def run():
            for _ in range(iters):
                fn()
    torch.cuda.synchronize()
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0.record()
    run()
    t1.record()
    torch.cuda.synchronize()
    us = t0.elapsed_time(t1) * 1e3 / iters
    return {"us_per_frame": round(us, 2), "bytes": moved, "GB_per_s": round(moved / us / 1e3, 1),
            "fraction_of_3.35TB_per_s": round(moved / (us * 1e-6) / HBM_BYTES_PER_S, 3), "sm_clock_after": sm_clock(),
            "timing": "CUDA graph of the launches" if graph else "launched from Python"}


def bench_kernels():
    from tecogan_b200 import kernels as K
    g = torch.Generator(device="cuda").manual_seed(1)
    res = {}
    for h, w in [(2160, 3840), (4320, 7680)]:
        src = torch.randint(0, 256, (h, w, 3), dtype=torch.uint8, device="cuda", generator=g)
        dst = torch.empty((3 * h // 2, w), dtype=torch.uint8, device="cuda")
        res["rgb_to_i420 %dx%d" % (h, w)] = timed(lambda: K.rgb_to_i420(src, dst), src.numel() + dst.numel())
    for h, w in [(540, 960), (1080, 1920)]:
        src = torch.randint(0, 256, (1, 3 * h // 2, w), dtype=torch.uint8, device="cuda", generator=g)
        out = torch.empty((1, h, w, 3), dtype=torch.uint8, device="cuda")
        res["i420_to_rgb %dx%d" % (h, w)] = timed(lambda: K.i420_to_rgb(src, out), src.numel() + out.numel())
        # the reader's two launches; bytes: I420 in, fp32 frame out (the uint8 frame between them is not counted)
        res["i420_to_rgb + frames_to_f32 %dx%d" % (h, w)] = timed(lambda: K.frames_to_f32(K.i420_to_rgb(src, out)),
                                                                  src.numel() + 4 * out.numel(), graph=False)
    for k, v in res.items():
        print("kernel %s: %s" % (k, json.dumps(v)), flush=True)
    return res


class HostI420Writer:
    """FrameWriter's interface with the conversion on the host: put() copies the RGB frame back to a pinned buffer on the
    producer's stream; the writer thread waits for it, runs cv2.cvtColor(COLOR_RGB2YUV_I420) and appends it to the
    sink."""

    def __init__(self, h, w, device, sink=None):
        self.sink, self.error = sink, None
        self.jobs, self.free, self.made = queue.Queue(), queue.Queue(), 0
        self.thread = threading.Thread(target=self._run, daemon=True)
        self.thread.start()

    def put(self, out_u8, path=None):
        if self.made < 3 and self.free.empty():
            self.made += 1
            self.free.put((torch.empty(out_u8.shape, dtype=torch.uint8, pin_memory=True), torch.cuda.Event()))
        slot = self.free.get()
        if isinstance(slot, BaseException):
            raise slot
        slot[0].copy_(out_u8, non_blocking=True)
        slot[1].record()
        self.jobs.put(slot)

    def _run(self):
        try:
            while True:
                item = self.jobs.get()
                if item is None:
                    return
                host, ev = item
                ev.synchronize()
                self.sink.write(cv2.cvtColor(host.numpy(), cv2.COLOR_RGB2YUV_I420))
                self.free.put((host, ev))
        except BaseException as e:
            self.error = e
            self.free.put(e)

    def close(self):
        self.jobs.put(None)
        self.thread.join()


def write_inputs(d, h, w, n, seed):
    """n seeded frames as PNG files and as one y4m stream of their I420."""
    from tecogan_b200 import y4m
    os.makedirs(d, exist_ok=True)
    g = np.random.default_rng(seed)
    base = PC.smooth(h, w + 2 * n, seed).astype(np.int64)
    with open(os.path.join(d, "in.y4m"), "wb") as y:
        y.write(y4m.format_header(w, h))
        for k in range(n):
            f = np.clip(base[:, 2 * k:2 * k + w] + g.integers(-3, 4, (h, w, 3)), 0, 255).astype(np.uint8)
            cv2.imwrite(os.path.join(d, "%04d.png" % (k + 1)), np.ascontiguousarray(f[:, :, ::-1]))
            y.write(b"FRAME\n" + cv2.cvtColor(f, cv2.COLOR_RGB2YUV_I420).tobytes())
    return d


def digest(path):
    h = hashlib.sha256()
    for n in sorted(os.listdir(path)) if os.path.isdir(path) else [path]:
        p = os.path.join(path, n) if os.path.isdir(path) else n
        h.update(os.path.basename(p).encode())
        with open(p, "rb") as f:
            h.update(f.read())
    return h.hexdigest()


def one_run(eng, d, out_dir, variant):
    import gc
    import main as M
    from tecogan_b200 import y4m
    from tecogan_b200.lib import writer as W
    from tecogan_b200.lib.dataloader import padded, stream_inputs
    os.makedirs(out_dir)
    eng.reset()                                   # every run starts the recurrence afresh, as a new command does
    gc.collect()
    torch.cuda.synchronize()
    real = W.FrameWriter
    if variant == "y4m_y4m_cv2_host":
        W.FrameWriter = HostI420Writer
    out = os.path.join(out_dir, "out.y4m")
    t0 = time.perf_counter()
    sink = None
    try:
        if variant == "png_jpeg":
            paths = sorted(os.path.join(d, f) for f in os.listdir(d) if f.endswith(".png"))
            frames, names = stream_inputs(paths, False), padded(paths)
        else:
            reader = y4m.Y4MReader(os.path.join(d, "in.y4m"))
            frames, names = reader.frames(), reader.names()
            sink = y4m.Y4MWriter(out, 4 * LR[1], 4 * LR[0])
        try:
            with contextlib.redirect_stdout(io.StringIO()):
                M.super_resolve_frames(eng, names, frames, out_dir, "output", "jpg", None, sink)
        finally:
            frames.close()
            if sink is not None:
                sink.close()
        torch.cuda.synchronize()
    finally:
        W.FrameWriter = real
    wall = time.perf_counter() - t0
    files = digest(out_dir if variant == "png_jpeg" else out)
    shutil.rmtree(out_dir)
    return wall, files


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
        raise SystemExit("bench_y4m: needs a CUDA device")
    res = {"card": card(), "cv2_threads": cv2.getNumThreads(), "command": {}}
    print("card:", res["card"], "| cv2 threads:", res["cv2_threads"], flush=True)
    res["kernel"] = bench_kernels()
    config.set_precision("bf16")
    M.load_checkpoint(V.set_default_store(V.VariableStore(seed=1)), "random:5", NRB)
    variants = ["y4m_y4m", "png_jpeg", "y4m_y4m_cv2_host"]
    with tempfile.TemporaryDirectory() as tmp:
        eng = InferenceEngine(LR[0], LR[1], NRB)
        warm = write_inputs(os.path.join(tmp, "warm"), LR[0], LR[1], 8, seed=7)
        for v in variants:                        # module loads, encoder plans, allocator
            one_run(eng, warm, os.path.join(tmp, "warm_" + v), v)
        d = write_inputs(os.path.join(tmp, "seq"), LR[0], LR[1], a.frames, seed=7)
        runs = {v: [] for v in variants}
        digests = {}
        for rep in range(a.reps):
            for v in variants:
                wall, files = one_run(eng, d, os.path.join(tmp, "out_%s_%d" % (v, rep)), v)
                digests.setdefault(v, set()).add(files)
                runs[v].append({"wall_s": round(wall, 3), "fps": round(a.frames / wall, 2), "sm_clock_after": sm_clock()})
                print("%s rep %d: %s" % (v, rep, json.dumps(runs[v][-1])), flush=True)
        res["command"] = {
            "frames": "%d x %dx%d -> %dx%d" % (a.frames, LR[0], LR[1], 4 * LR[0], 4 * LR[1]),
            "runs": runs,
            "y4m_outputs_identical": len(digests["y4m_y4m"] | digests["y4m_y4m_cv2_host"]) == 1,
            "each_variant_repeatable": all(len(v) == 1 for v in digests.values())}
        print("command: %s" % json.dumps(res["command"]), flush=True)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
