"""Training input from disk: the host loader (HRClipLoader) against the device frame store (FrameStore), and what each
does to the bf16 training step.  Generates seeded PNG scenes (smooth noise, half at 960x540 and half at 640x360, 120
frames each) in a temporary directory and reports, in one JSON line with the GPU's name and power limit and the host's
core count:
  * host-loader ms per batch (HRClipLoader.batches, B=4 x 10 frames, crop 32) at queue_thread 6 and 12;
  * store build time and bytes, store ms per batch (FrameStore.batch, synchronised; and the batches() iterator);
  * bf16 FRVSR and TecoGAN ms per training step fed from disk through each path, against main.py's --synthetic_data
    batches and against a step on resident inputs.

    python tools/bench_loader.py [--scenes 4] [--steps 30] [--out result.json]"""
import argparse
import concurrent.futures
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
from tecogan_b200 import config, variables as V  # noqa: E402
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scenes", type=int, default=4)
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    dev = torch.device("cuda")
    n, w = args.steps, args.warmup
    res = {"gpu": gpu_info(), "host_cores": os.cpu_count(), "scenes": args.scenes, "frame_sizes": ["%dx%d" % (b, a) for a, b in SIZES],
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
            step = iter(range(10 ** 9))
            feeds = {
                "resident": lambda: Net.train(),
                "synthetic_data": lambda: Net.train(*frvsr_gpu_data_loader(M.synthetic_hr_batch(F, next(step), 0, dev), F)),
                "host_loader_q6": lambda: Net.train(*frvsr_gpu_data_loader(next(host_it).to(dev, non_blocking=True), F)),
                "frame_store": lambda: Net.train(*frvsr_gpu_data_loader(next(store_it), F)),
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
            res[name] = out
            host_it.close()
            store_it.close()
            del Net
            torch.cuda.empty_cache()
    finally:
        shutil.rmtree(work, ignore_errors=True)
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
