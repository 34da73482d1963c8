"""Cost of training monitoring (main.py --mode train --summary_dir) at the benchmarked training shapes, bf16 training:
ms per Network.train() step, per Network.train.evaluate() (the validation pass, one batch of the same shape) and per
10-frame test-sequence pass (main.test_while_train on 144x180 calendar frames, PNG writes included), and what one
validation pass or one test-sequence pass adds to 100 training steps.  Prints one JSON line, with the GPU's name and
power limit read in the same run.

    python tools/bench_validation.py [--steps 20] [--out result.json]"""
import argparse
import json
import os
import subprocess
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
from tecogan_b200.lib.dataloader import frvsr_gpu_data_loader  # noqa: E402
from tecogan_b200.lib.Teco import FRVSR, TecoGAN  # noqa: E402

COMMON = ["--mode", "train", "--batch_size", "4", "--RNN_N", "10", "--crop_size", "32", "--learning_rate", "0.00005",
          "--decay_rate", "1.0", "--stair", "--beta", "0.9", "--precision", "bf16"]
CASES = {   # bench.py's training workloads (runGan.py case 4 / case 3 flags)
    "config3_frvsr": ["--num_resblock", "10", "--ratio", "-0.01", "--nopingpang"],
    "config4_tecogan": ["--num_resblock", "16", "--ratio", "0.01", "--pingpang", "--pp_scaling", "0.5", "--vgg_scaling", "0.2",
                        "--Dt_mergeDs", "--D_LAYERLOSS"],
}


def ev_ms(fn, n):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(n):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / n


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    dev = torch.device("cuda")
    config.set_train_precision("bf16")
    res = {"gpu": gpu_info(), "train_precision": "bf16", "steps": args.steps}
    work = tempfile.mkdtemp(prefix="teco_bench_val_")
    import cv2
    cal = np.load(os.path.join(ROOT, "tests", "golden", "calendar_lr.npz"))["full_u8"]
    os.makedirs(os.path.join(work, "LR", "calendar"))
    for i in range(10):
        cv2.imwrite(os.path.join(work, "LR", "calendar", "%04d.png" % (i + 1)), cal[min(i, len(cal) - 1)][:, :, ::-1])
    for name, extra in CASES.items():
        F = M.parse_flags(COMMON + extra + ["--output_dir", os.path.join(work, name)])
        os.makedirs(F.output_dir, exist_ok=True)
        gan = F.ratio > 0
        st = V.set_default_store(V.VariableStore())
        st.load(xavier_params(1, F.num_resblock, gan, F.vgg_scaling > 0))
        lr, tg = frvsr_gpu_data_loader(M.synthetic_hr_batch(F, 0, 0, dev), F)
        vlr, vtg = frvsr_gpu_data_loader(M.synthetic_hr_batch(F, 0, 0, dev, validation=True), F)
        Net = TecoGAN(lr, tg, F) if gan else FRVSR(lr, tg, F)
        for _ in range(3):
            Net.train()
            Net.train.evaluate(vlr, vtg)
        torch.cuda.synchronize()
        n = args.steps
        # alternate the two measurements so that both see the same state of a shared machine
        t_train, t_eval = [], []
        for _ in range(3):
            t_train.append(ev_ms(lambda: Net.train(), n))
            t_eval.append(ev_ms(lambda: Net.train.evaluate(vlr, vtg), n))
        cwd = os.getcwd()
        os.chdir(work)
        try:
            with open(os.devnull, "w") as null:
                so, sys.stdout = sys.stdout, null
                try:
                    M.test_while_train(F, 0)                       # warm-up: module loads, graph capture
                    t_seq = []
                    for k in range(3):
                        torch.cuda.synchronize()
                        t0 = time.perf_counter()
                        M.test_while_train(F, k + 1)
                        t_seq.append((time.perf_counter() - t0) * 1e3)
                finally:
                    sys.stdout = so
        finally:
            os.chdir(cwd)
        ms_train, ms_eval, ms_seq = float(np.median(t_train)), float(np.median(t_eval)), float(np.median(t_seq))
        res[name] = {"ms_per_train_step": ms_train, "ms_per_evaluate": ms_eval, "ms_per_test_sequence": ms_seq,
                     "spread_train_ms": [min(t_train), max(t_train)], "spread_evaluate_ms": [min(t_eval), max(t_eval)],
                     "spread_test_sequence_ms": [min(t_seq), max(t_seq)],
                     "validation_pass_added_per_100_steps_pct": 100.0 * ms_eval / (100.0 * ms_train),
                     "test_sequence_added_per_100_steps_pct": 100.0 * ms_seq / (100.0 * ms_train)}
        del Net
        torch.cuda.empty_cache()
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
