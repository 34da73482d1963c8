"""PNG decode on the device (tecogan_b200.png.decode_png) against cv2.imread on the host, and the two callers built on it.

  python tools/bench_png_decode.py [--reps 3] [--out results/bench_png_decode.json]

Prints the card's name and power limit, then:
  * per frame size (576x720, 1080x1920, 2160x3840; seeded smooth frames with noise, written by cv2.imwrite): the three
    kernels of one batch (CUDA events around teco_png_decode_rgb8 alone, inputs already staged on the device), decode_png end to end with
    the file reads (6 host threads), and cv2.imread on one thread and on a 6-thread pool -- alternated in each rep;
  * a FrameStore build over ~540 MB of 576x720 scenes, and of 1080x1920 scenes, against the host-decoded build of the
    same scenes (6 threads);
  * metrics.py on a seeded 41-frame 576x720 folder pair and a 12-frame 2160x3840 one, with and without --tof, device
    decoding against read_rgb.
Every comparison first checks that the bytes (or the written metrics files) are identical.  Temporary files only.
"""
import argparse
import concurrent.futures
import hashlib
import json
import os
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

SIZES = {(576, 720): 64, (1080, 1920): 24, (2160, 3840): 8}     # frames per batch


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip()


def frame(h, w, seed):
    g = np.random.default_rng(seed)
    f = PC.smooth(h, w, seed).astype(np.int64) + g.integers(-3, 4, (h, w, 3))
    return np.clip(f, 0, 255).astype(np.uint8)


def write_frames(d, h, w, n, seed0=0):
    os.makedirs(d, exist_ok=True)
    base = frame(h, w, seed0)
    paths = []
    for k in range(n):
        p = os.path.join(d, "%04d.png" % k)
        cv2.imwrite(p, np.ascontiguousarray(np.roll(base, 3 * k, axis=1)[:, :, ::-1]))
        paths.append(p)
    return paths


def cv2_rgb(p):
    return np.ascontiguousarray(cv2.imread(p, cv2.IMREAD_COLOR)[:, :, ::-1])


def timed(fn):
    torch.cuda.synchronize()
    t = time.perf_counter()
    r = fn()
    torch.cuda.synchronize()
    return r, (time.perf_counter() - t) * 1e3


def bench_sizes(tmp, reps):
    from tecogan_b200 import png as P
    out = {}
    pool = concurrent.futures.ThreadPoolExecutor(6)
    for (h, w), n in SIZES.items():
        paths = write_frames(os.path.join(tmp, "%dx%d" % (h, w)), h, w, n, seed0=h)
        ref = [cv2_rgb(p) for p in paths]
        got = P.decode_png(paths, threads=6)
        assert all(np.array_equal(g.cpu().numpy(), r) for g, r in zip(got, ref)), (h, w)
        streams = [P.load_png(p) for p in paths]
        assert all(s is not None for s in streams)
        dst = torch.empty(n * h * w * 3, dtype=torch.uint8, device="cuda")
        items = [(s, k * h * w * 3) for k, s in enumerate(streams)]
        assert not P.decode_streams(items, dst).any()
        assert np.array_equal(dst.cpu().numpy(), np.concatenate([r.reshape(-1) for r in ref]))
        rows = {"device_kernel_ms": [], "decode_png_ms": [], "cv2_1t_ms": [], "cv2_6t_ms": []}
        for _ in range(reps):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            ws_need = [P.decode_plan_bytes(s.h, s.w, s.colour, s.depth) for s in streams]
            args = P.stage_batch(items, ws_need, sum(ws_need), dst)
            torch.cuda.synchronize()
            e0.record()                               # the three kernels alone: staging and copies are outside
            P.launch_batch(*args)
            e1.record()
            torch.cuda.synchronize()
            assert not args[-1].any()
            rows["device_kernel_ms"].append(e0.elapsed_time(e1))
            rows["decode_png_ms"].append(timed(lambda: P.decode_png(paths, threads=6))[1])
            rows["cv2_1t_ms"].append(timed(lambda: [cv2_rgb(p) for p in paths])[1])
            rows["cv2_6t_ms"].append(timed(lambda: list(pool.map(cv2_rgb, paths)))[1])
        med = {k: float(np.median(v)) for k, v in rows.items()}
        med.update(frames=n, mb_decoded=n * h * w * 3 / 1e6, mb_files=sum(os.path.getsize(p) for p in paths) / 1e6)
        med.update({k.replace("_ms", "_ms_per_frame"): med[k] / n for k in rows})
        out["%dx%d" % (h, w)] = med
        print("%dx%d x%d: %s" % (h, w, n, json.dumps({k: round(v, 3) for k, v in med.items()})), flush=True)
    pool.shutdown()
    return out


def host_store(store_cls, loaders, threads):
    """The host-decoded build: every frame decoded by cv2 on `threads` threads into a pinned stage, copied up per
    256 MiB chunk (FrameStore's build before the device decoder)."""
    s = object.__new__(store_cls)
    L = loaders[0]
    paths = [L.frame_path(ci, f) for ci in range(len(L.clips)) for f in range(L.F.max_frm + 1)]
    hw = np.array([L.frame_size(p) for p in paths], np.int64)
    off = np.concatenate([[0], np.cumsum(hw[:, 0] * hw[:, 1] * 3)]).astype(np.int64)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    buf = torch.empty(int(off[-1]), dtype=torch.uint8, device="cuda")
    stage = torch.empty(min(int(off[-1]), 256 << 20), dtype=torch.uint8).pin_memory()
    host = stage.numpy()
    with concurrent.futures.ThreadPoolExecutor(threads) as pool:
        i = 0
        while i < len(paths):
            j = i + 1
            while j < len(paths) and off[j + 1] - off[i] <= stage.numel():
                j += 1

            def put(k, i=i):
                host[off[k] - off[i]:off[k + 1] - off[i]] = L.decode(paths[k]).reshape(-1)
            list(pool.map(put, range(i, j)))
            buf[int(off[i]):int(off[j])].copy_(stage[:int(off[j] - off[i])])
            i = j
    torch.cuda.synchronize()
    s.buf = buf
    return s, (time.perf_counter() - t0) * 1e3


def bench_store(tmp, reps, h, w, scenes, frames):
    from tests.test_dataloader_host import Flags
    from tecogan_b200.lib.dataloader import FrameStore, HRClipLoader
    root = os.path.join(tmp, "store_%dx%d" % (h, w))
    for sidx in range(scenes):
        d = os.path.join(root, "scene_%04d" % (2000 + sidx))
        for k, p in enumerate(write_frames(d, h, w, frames, seed0=sidx)):
            os.rename(p, os.path.join(d, "col_high_%04d.png" % k))
    F = Flags(input_video_dir=root, str_dir=2000, end_dir=2000 + scenes - 1, max_frm=frames - 1, RNN_N=4, batch_size=2,
              crop_size=32, queue_thread=6)
    L = HRClipLoader(F)
    dev_ms, host_ms = [], []
    for _ in range(reps):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        st = FrameStore([L], "cuda")
        torch.cuda.synchronize()
        dev_ms.append((time.perf_counter() - t0) * 1e3)
        hs, ms = host_store(FrameStore, [L], 6)
        host_ms.append(ms)
        same = hashlib.sha256(st.buf.cpu().numpy().tobytes()).hexdigest() == hashlib.sha256(hs.buf.cpu().numpy().tobytes()).hexdigest()
        assert same
        nbytes = st.nbytes
        del st, hs
        torch.cuda.empty_cache()
    r = {"frame": "%dx%d" % (h, w), "store_mb": nbytes / 1e6, "frames": scenes * frames, "device_build_ms": float(np.median(dev_ms)),
         "host_build_6t_ms": float(np.median(host_ms)), "identical": True}
    print("frame store: %s" % json.dumps(r), flush=True)
    return r


def bench_metrics(tmp, reps, h, w, n):
    import metrics as CLI
    tmp = os.path.join(tmp, "metrics_%dx%d" % (h, w))
    write_frames(os.path.join(tmp, "m_res"), h, w, n, seed0=7)
    write_frames(os.path.join(tmp, "m_tar"), h, w, n, seed0=8)
    host_read = lambda paths: [torch.from_numpy(CLI.read_rgb(p)).cuda() for p in paths]
    device_read = CLI.read_folder
    out = {}
    for tof in (False, True):
        args = ["--results", os.path.join(tmp, "m_res"), "--targets", os.path.join(tmp, "m_tar")] + (["--tof"] if tof else [])
        dev_ms, host_ms = [], []
        for r in range(reps + 1):                     # the first round warms both paths
            for name, fn, acc in (("dev", device_read, dev_ms), ("host", host_read, host_ms)):
                CLI.read_folder = fn
                logd = os.path.join(tmp, "log_%s_%d_%d" % (name, tof, r))
                _, ms = timed(lambda: CLI.main(["--output", logd] + args))
                if r:
                    acc.append(ms)
            for f in ("metricsfile.txt", "metrics.csv"):
                a = open(os.path.join(tmp, "log_dev_%d_%d" % (tof, r), f)).read()
                assert a == open(os.path.join(tmp, "log_host_%d_%d" % (tof, r), f)).read(), f
        CLI.read_folder = device_read
        out["tof" if tof else "plain"] = {"device_ms": float(np.median(dev_ms)), "read_rgb_ms": float(np.median(host_ms)),
                                          "identical": True}
        print("metrics.py%s, %d frames of %dx%d: %s" % (" --tof" if tof else "", n, h, w,
                                                         json.dumps(out["tof" if tof else "plain"])), flush=True)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "bench_png_decode needs a GPU"
    res = {"card": card()}
    print("card:", res["card"], flush=True)
    with tempfile.TemporaryDirectory() as tmp:
        res["sizes"] = bench_sizes(tmp, a.reps)
        res["frame_store"] = bench_store(tmp, a.reps, 576, 720, 36, 12)          # 432 frames: 537 MB
        res["frame_store_1080p"] = bench_store(tmp, a.reps, 1080, 1920, 8, 11)   # 88 frames: 547 MB
        res["metrics"] = bench_metrics(tmp, a.reps, 576, 720, 41)
        res["metrics_4k"] = bench_metrics(tmp, a.reps, 2160, 3840, 12)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
