"""Training input from disk: the host loader (HRClipLoader) against the device frame store (FrameStore), and what each
does to the bf16 training step.  Generates seeded PNG scenes (smooth noise, half at 960x540 and half at 640x360, 120
frames each) in a temporary directory and reports, in one JSON line with the GPU's name and power limit and the host's
core count:
  * host-loader ms per batch (HRClipLoader.batches, B=4 x 10 frames, crop 32) at queue_thread 6 and 12;
  * store build time and bytes, store ms per batch (FrameStore.batch, synchronised; and the batches() iterator);
  * the same for the store in host memory (FrameStore(placement='host')), and the gather per batch in us (CUDA events)
    of teco_gather_clips_host_u8 and of teco_gather_clips_u8 pointed at the same mapped store, over random windows;
  * bf16 FRVSR and TecoGAN ms per training step fed from disk through each path, against main.py's --synthetic_data
    batches and against a step on resident inputs;
  * the host's MemTotal and the room tecogan_b200/hostmem.py::host_room_bytes leaves for a host store;
  * with --mapped_gib G, the same two gathers over a registered mapping of G GiB (960x540 frames back to back, each
    window in a random frame anywhere in it), against the same draws confined to the first 0.5 GiB: whether windows
    spread over tens of GiB of mapped memory cost more than over a small store (the GPU's translation of system
    addresses).  Writing and decoding PNG scenes of that size is not needed to measure the gather.

    python tools/bench_loader.py [--scenes 4] [--steps 30] [--mapped_gib 64] [--out result.json]"""
import argparse
import concurrent.futures
import ctypes
import json
import os
import shutil
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import main as M  # noqa: E402
from tecogan_b200 import _ffi, config, kernels as K, variables as V  # noqa: E402
from tecogan_b200.hostmem import HostMapping, host_room_bytes  # noqa: E402
from tecogan_b200.init_params import xavier_params  # noqa: E402
from tecogan_b200.lib.dataloader import FrameStore, HRClipLoader, frvsr_gpu_data_loader  # noqa: E402
from tecogan_b200.lib.Teco import FRVSR, TecoGAN  # noqa: E402
from tools.bench_validation import CASES, COMMON, gpu_info  # noqa: E402

SIZES = ((540, 960), (360, 640))


def write_scenes(root, scenes, frames):
    """Scenes 2000.. alternating between the two sizes; frame f of a scene is a seeded smooth field shifted by f pixels."""
    import cv2

    def scene(i):
        h, w = SIZES[i % 2]
        rng = np.random.default_rng(1000 + i)
        base = cv2.resize(rng.integers(0, 256, ((h + frames) // 16 + 2, (w + 2 * frames) // 16 + 2, 3), dtype=np.uint8),
                          None, fx=16, fy=16, interpolation=cv2.INTER_CUBIC)
        d = os.path.join(root, "scene_%04d" % (2000 + i))
        os.makedirs(d)
        for f in range(frames):
            cv2.imwrite(os.path.join(d, "col_high_%04d.png" % f), np.ascontiguousarray(base[f:f + h, 2 * f:2 * f + w]))
    with concurrent.futures.ThreadPoolExecutor(max_workers=os.cpu_count()) as pool:
        list(pool.map(scene, range(scenes)))


def wall_ms(fn, n):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(n):
        fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3 / n


def gather_us(store, n, rounds=5):
    """us per batch of teco_gather_clips_host_u8 and of teco_gather_clips_u8 reading the same mapped host store, over the
    windows of n different batches (CUDA events around each kernel's n launches, median of `rounds`, alternating)."""
    tables = [torch.from_numpy(store.table(k)).cuda() for k in range(n)]
    return time_gathers(store._host.dev_addr, tables, store.loader.tar_size, rounds)


def mapped_gather_us(gib, n=200, S=136, windows=40, rounds=5):
    """gather_us over a registered mapping of `gib` GiB holding 960x540 frames back to back: n batches of `windows`
    random windows (random frame, origin and flip), once over every frame of the mapping and once over the frames of its
    first 0.5 GiB."""
    H, W = 540, 960
    fb = H * W * 3
    m = HostMapping.create(int(gib * 2 ** 30))
    m.close_fd()
    try:
        t0 = time.time()
        m.register()
        res = {"mapped_gib": gib, "mapped_register_s": time.time() - t0}
        rng = np.random.default_rng(5)
        for key, frames in (("all", m.nbytes // fb), ("first_0.5gib", (2 ** 29) // fb)):
            tables = []
            for _ in range(n):
                f = rng.integers(0, frames, windows)
                y, x = rng.integers(0, H - S + 1, windows), rng.integers(0, W - S + 1, windows)
                tables.append(torch.from_numpy(np.stack([f * fb + (y * W + x) * 3, np.full(windows, 3 * W),
                                                         rng.integers(0, 2, windows)], 1).astype(np.int64)).cuda())
            res[key] = time_gathers(m.dev_addr, tables, S, rounds)
        return res
    finally:
        m.close()


def time_gathers(addr, tables, S, rounds):
    n = len(tables)
    out = torch.empty((tables[0].shape[0], S, S, 3), device="cuda")

    def new(t):
        K.gather_clips_host_u8(addr, t, S)

    def old(t):
        _ffi.call("teco_gather_clips_u8", ctypes.c_void_p(addr), _ffi.ptr(t, torch.int64), t.shape[0], S,
                  _ffi.ptr(out, torch.float32), _ffi.stream_ptr())
    ref = K.gather_clips_host_u8(addr, tables[0], S)
    old(tables[0])
    assert torch.equal(ref, out), "the two kernels disagree on the mapped store"
    res = {"gather_host_kernel_us": [], "gather_u8_kernel_on_mapped_us": []}
    for _ in range(rounds):
        for key, fn in (("gather_host_kernel_us", new), ("gather_u8_kernel_on_mapped_us", old)):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            for t in tables:
                fn(t)
            b.record()
            b.synchronize()
            res[key].append(a.elapsed_time(b) * 1e3 / n)
    return {k: float(np.median(v)) for k, v in res.items()} | {"spread_" + k: [min(v), max(v)] for k, v in res.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scenes", type=int, default=4)
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--mapped_gib", type=float, default=0)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    dev = torch.device("cuda")
    n, w = args.steps, args.warmup
    meminfo = dict(l.split(":", 1) for l in open("/proc/meminfo").read().splitlines() if ":" in l)
    res = {"gpu": gpu_info(), "host_cores": os.cpu_count(), "host_mem_total": meminfo["MemTotal"].strip(),
           "host_room_gib": host_room_bytes() / 2 ** 30, "scenes": args.scenes, "frame_sizes": ["%dx%d" % (b, a) for a, b in SIZES],
           "batch": "B=4 x 10 frames, crop 32 (136x136 HR windows)", "steps": n}
    work = tempfile.mkdtemp(prefix="teco_bench_loader_")
    try:
        t0 = time.time()
        write_scenes(work, args.scenes, 120)
        res["scene_write_s"] = round(time.time() - t0, 1)
        data = ["--input_video_dir", work, "--str_dir", "2000", "--end_dir", str(2000 + args.scenes - 1), "--max_frm", "119"]
        F0 = M.parse_flags(COMMON + data + ["--output_dir", work])

        for qt in (6, 12):
            it = HRClipLoader(F0, queue_thread=qt).batches()
            for _ in range(w):
                next(it)
            t0 = time.perf_counter()
            for _ in range(n):
                next(it)
            res["host_loader_ms_per_batch_q%d" % qt] = (time.perf_counter() - t0) * 1e3 / n
            it.close()

        L = HRClipLoader(F0)
        store = FrameStore([L], dev)
        res["store_bytes"] = store.nbytes
        res["store_frames"] = len(store.paths)
        res["store_build_s"] = store.build_seconds
        res["store_build_threads"] = L.queue_thread
        k = iter(range(10 ** 9))
        res["store_ms_per_batch"] = wall_ms(lambda: store.batch(next(k)), n)
        it = store.batches()
        res["store_iter_ms_per_batch"] = wall_ms(lambda: next(it), n)
        it.close()
        same = all(torch.equal(store.batch(s), L.batch(s).to(dev)) for s in range(3))
        res["store_equals_host_loader_first_3_batches"] = same

        hstore = FrameStore([L], dev, placement="host")
        res["host_store_bytes"] = hstore.nbytes
        res["host_store_build_s"] = hstore.build_seconds
        k = iter(range(10 ** 9))
        res["host_store_ms_per_batch"] = wall_ms(lambda: hstore.batch(next(k)), n)
        it = hstore.batches()
        res["host_store_iter_ms_per_batch"] = wall_ms(lambda: next(it), n)
        it.close()
        res["host_store_equals_store_first_3_batches"] = all(torch.equal(hstore.batch(s), store.batch(s)) for s in range(3))
        res.update(gather_us(hstore, 200))

        config.set_train_precision("bf16")
        for name, extra in CASES.items():
            F = M.parse_flags(COMMON + extra + data + ["--output_dir", work])
            gan = F.ratio > 0
            V.set_default_store(V.VariableStore()).load(xavier_params(1, F.num_resblock, gan, F.vgg_scaling > 0))
            lr0, tg0 = frvsr_gpu_data_loader(M.synthetic_hr_batch(F, 0, 0, dev), F)
            Net = TecoGAN(lr0, tg0, F) if gan else FRVSR(lr0, tg0, F)
            for _ in range(3):
                Net.train()
            host_it = HRClipLoader(F).batches()
            store_it = store.batches()
            hstore_it = hstore.batches()
            step = iter(range(10 ** 9))
            feeds = {
                "resident": lambda: Net.train(),
                "synthetic_data": lambda: Net.train(*frvsr_gpu_data_loader(M.synthetic_hr_batch(F, next(step), 0, dev), F)),
                "host_loader_q6": lambda: Net.train(*frvsr_gpu_data_loader(next(host_it).to(dev, non_blocking=True), F)),
                "frame_store": lambda: Net.train(*frvsr_gpu_data_loader(next(store_it), F)),
                "host_store": lambda: Net.train(*frvsr_gpu_data_loader(next(hstore_it), F)),
            }
            r = {key: [] for key in feeds}
            for key, fn in feeds.items():
                wall_ms(fn, w)
            for _ in range(3):                  # alternate the feeds so that all of them see the same state of the machine
                for key, fn in feeds.items():
                    r[key].append(wall_ms(fn, n))
            out = {"ms_per_step_" + key: float(np.median(v)) for key, v in r.items()}
            out.update({"spread_" + key: [min(v), max(v)] for key, v in r.items()})
            out["frame_store_vs_synthetic_pct"] = 100.0 * (out["ms_per_step_frame_store"] / out["ms_per_step_synthetic_data"] - 1)
            out["host_store_vs_frame_store_pct"] = 100.0 * (out["ms_per_step_host_store"] / out["ms_per_step_frame_store"] - 1)
            res[name] = out
            host_it.close()
            store_it.close()
            hstore_it.close()
            del Net
            torch.cuda.empty_cache()
        hstore.close()
    finally:
        shutil.rmtree(work, ignore_errors=True)
    if args.mapped_gib > 0:
        res["mapped_store"] = mapped_gather_us(args.mapped_gib)
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
