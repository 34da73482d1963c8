"""Cost of deterministic training: FRVSR (config 3: case 4, 10 blocks) and TecoGAN (config 4: case 3, 16 blocks, ping-pong,
VGG) training steps at B=4, RNN_N=10, 32x32 LR, in bf16 and fp32, with the default atomic reductions and with
--deterministic, timed alternately in one process (rounds of `steps` CUDA-graph steps per mode) so both modes see the same
machine state.  Prints the card and its power limit beside the numbers.

    python tools/bench_deterministic.py [steps per round] [rounds]
"""
import os
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import main as M  # noqa: E402
from tecogan_b200 import config  # noqa: E402
from tecogan_b200 import variables as V  # noqa: E402
from tecogan_b200.init_params import xavier_params  # noqa: E402
from tecogan_b200.lib.dataloader import frvsr_gpu_data_loader  # noqa: E402
from tecogan_b200.lib.Teco import FRVSR, TecoGAN  # noqa: E402

FLAGS = {
    "frvsr": ["--num_resblock", "10", "--ratio", "-0.01", "--nopingpang"],
    "tecogan": ["--num_resblock", "16", "--ratio", "0.01", "--pingpang", "--pp_scaling", "0.5", "--vgg_scaling", "0.2"],
}


def make_net(which, precision, det):
    """A trainer whose CUDA graph is captured with the kernels of `det` (the mode is read while the step is recorded)."""
    F = M.parse_flags(["--mode", "train", "--output_dir", "/tmp/unused", "--learning_rate", "0.00005", "--decay_rate", "1.0",
                       "--stair"] + FLAGS[which])
    config.set_train_precision(precision)
    config.set_deterministic(det)
    st = V.set_default_store(V.VariableStore())
    gan = F.ratio > 0
    st.load(xavier_params(1, F.num_resblock, gan, F.vgg_scaling > 0))
    lr, tg = frvsr_gpu_data_loader(M.synthetic_hr_batch(F, 0, 0, torch.device("cuda")), F)
    net = TecoGAN(lr, tg, F) if gan else FRVSR(lr, tg, F)
    for _ in range(2):
        net.train()
    torch.cuda.synchronize()
    return st, net


def timed(st, net, steps):
    V.set_default_store(st)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(steps):
        net.train()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) / steps * 1e3


def main():
    steps = int(sys.argv[1]) if len(sys.argv) > 1 else 20
    rounds = int(sys.argv[2]) if len(sys.argv) > 2 else 5
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip()
    print("device: %s (name, power limit, max SM clock)" % q)
    for which in ("frvsr", "tecogan"):
        for precision in ("bf16", "fp32"):
            nets = {det: make_net(which, precision, det) for det in (False, True)}
            times = {False: [], True: []}
            for _ in range(rounds):
                for det in (False, True):
                    times[det].append(timed(*nets[det], steps))
            med = {d: sorted(t)[len(t) // 2] for d, t in times.items()}
            print("%-8s %-5s default %7.2f ms/step [%s]   deterministic %7.2f ms/step [%s]   cost %+.1f %%" % (
                which, precision, med[False], " ".join("%.2f" % t for t in times[False]), med[True],
                " ".join("%.2f" % t for t in times[True]), 100.0 * (med[True] / med[False] - 1.0)))
            del nets
            torch.cuda.empty_cache()
    config.set_deterministic(False)


if __name__ == "__main__":
    main()
