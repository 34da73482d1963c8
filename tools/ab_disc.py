"""Device time of the discriminator's four 4x4 stride-2 convolutions (disblock_1/3/5/7) on the fp32 CUDA-core kernels and on
the tensor-core space-to-depth path of bf16 training, and of a whole bf16 TecoGAN step with either.

  python tools/ab_disc.py [--out DIR] [--no-step]

Shapes are those of the TecoGAN training step at B = 4, RNN_N = 10 with ping-pong (t_batch = 24 triplets of 128 x 128 HR
crops, a real and a fake call: 48 samples per layer).  Per layer, forward, input gradient and weight gradient are timed
alone in CUDA-graph replay with CUDA events (REPS calls per graph, the median of ROUNDS replays):
  fp32     conv2d_f32_kernel; four phase launches of it for the input gradient; conv2d_wgrad_f32_kernel
  tc       teco_f32_to_bf16_s2d2 + teco_conv4x4s2_tc + bf16 -> fp32; fp32 -> bf16 dz + teco_conv4x4s2_dgrad_tc +
           teco_bf16_d2s2_to_f32; teco_conv3x3_wgrad_tc over all 36 (tap, phase) slots + the 16 live slots' index_select
           (the weight packing, once per step, is timed with the forward)
TFLOP/s counts the live MACs only (N * OH * OW * 16 * Cin * Cout per pass).  Then, unless --no-step, a bf16 TecoGAN step
is timed with the disblocks on each path (three alternating rounds of STEPS graph-replayed steps), and one torch.profiler
pass of the fp32-disblock step gives the share of the fp32 convolution kernels in its device time.  Prints the card and its
power limit; DIR/ab_disc.json gets the same numbers."""
import argparse
import contextlib
import json
import os
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from tecogan_b200 import config, kernels as K  # noqa: E402
from tecogan_b200._ffi import call, ptr, stream_ptr  # noqa: E402

REPS, ROUNDS, STEPS = 20, 7, 10
N = 48
LAYERS = [("disblock_1", 128, 64, 64), ("disblock_3", 64, 64, 64), ("disblock_5", 32, 64, 128), ("disblock_7", 16, 128, 256)]


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name(0)


def graph_us(fn):
    """Median device microseconds of one fn() over ROUNDS replays of a graph holding REPS calls."""
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        fn()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=s):
            for _ in range(REPS):
                fn()
    torch.cuda.current_stream().wait_stream(s)
    g.replay()
    torch.cuda.synchronize()
    ts = []
    for _ in range(ROUNDS):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        g.replay()
        e1.record()
        torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1) * 1000.0 / REPS)
    return sorted(ts)[len(ts) // 2]


def layer_rows():
    rows = []
    g = torch.Generator(device="cuda").manual_seed(0)
    for name, H, cin, cout in LAYERS:
        h = H // 2
        x = torch.randn(N, H, H, cin, device="cuda", generator=g)
        w = torch.randn(4, 4, cin, cout, device="cuda", generator=g) * 0.05
        dz = torch.randn(N, h, h, cout, device="cuda", generator=g)
        y, dx, dw = torch.empty(N, h, h, cout, device="cuda"), torch.empty_like(x), torch.empty_like(w)
        xs = torch.empty(N, h, h, 4 * cin, device="cuda", dtype=torch.bfloat16)
        ys = torch.empty(N, h, h, cout, device="cuda", dtype=torch.bfloat16)
        dxs = torch.empty_like(xs)
        dwp = torch.empty(3, 3, 4 * cin, cout, device="cuda")
        K.tc_cache_clear()
        wpk, wpk_t = K._c4s2_packed(w, 0), K._c4s2_packed(w, 1)
        idx = K._c4s2_index(w.device)

        def tc_fwd():
            call("teco_pack_conv4x4s2_bf16", ptr(w), cin, cout, 0, ptr(wpk), stream_ptr())
            call("teco_f32_to_bf16_s2d2", ptr(x), ptr(xs), N, H, H, cin, stream_ptr())
            call("teco_conv4x4s2_tc", N, H, H, cin, cout, 0, ptr(xs), ptr(wpk), ptr(None), ptr(ys), stream_ptr())
            K._from_bf16_rows(ys, cout)

        def tc_dgrad():
            call("teco_pack_conv4x4s2_bf16", ptr(w), cin, cout, 1, ptr(wpk_t), stream_ptr())
            dzb = K._to_bf16_rows(dz, cout)
            call("teco_conv4x4s2_dgrad_tc", N, H, H, cin, cout, ptr(dzb), ptr(wpk_t), ptr(dxs), stream_ptr())
            call("teco_bf16_d2s2_to_f32", ptr(dxs), ptr(dx), N, H, H, cin, stream_ptr())

        dzb0 = K._to_bf16_rows(dz, cout)

        def tc_wgrad():
            K.conv3x3_wgrad_tc(xs, dzb0, dwp, 4 * cin, cout)
            dwp.view(36, cin, cout).index_select(0, idx)

        fp32 = {
            "fwd": lambda: K.conv2d_raw(x, w, None, y, stride=2, pad_t=1, pad_l=1, OH=h, OW=h),
            "dgrad": lambda: K.conv_transpose2x_raw(dz, w, None, dx, pad=1),
            "wgrad": lambda: K.conv2d_wgrad_raw(x, dz, dw, None, stride=2, pad_t=1, pad_l=1, OH=h, OW=h),
        }
        tc = {"fwd": tc_fwd, "dgrad": tc_dgrad, "wgrad": tc_wgrad}
        mac = N * h * h * 16 * cin * cout
        row = {"layer": name, "out": h, "cin": cin, "cout": cout, "live_gmac": mac / 1e9}
        for var, fns in (("fp32", fp32), ("tc", tc)):
            for op, fn in fns.items():
                us = graph_us(fn)
                row["%s_%s_us" % (var, op)] = us
                row["%s_%s_tflops" % (var, op)] = 2.0 * mac / (us * 1e-6) / 1e12
        rows.append(row)
    return rows


def make_net(tc_disc):
    """A bf16 TecoGAN training step at the benchmark's config (tools/bench_train.py), with the disblocks on the tensor
    cores or on the fp32 kernels."""
    import main as M
    from tecogan_b200 import variables as V
    from tecogan_b200.init_params import xavier_params
    from tecogan_b200.lib.dataloader import frvsr_gpu_data_loader
    from tecogan_b200.lib.Teco import TecoGAN
    F = M.parse_flags(["--mode", "train", "--output_dir", "/tmp/x", "--num_resblock", "16", "--ratio", "0.01", "--pingpang",
                       "--pp_scaling", "0.5", "--vgg_scaling", "0.2", "--learning_rate", "0.00005", "--decay_rate", "1.0",
                       "--stair"])
    config.set_train_precision("bf16")
    V.set_default_store(V.VariableStore()).load(xavier_params(1, F.num_resblock, True, True))
    lr, tg = frvsr_gpu_data_loader(M.synthetic_hr_batch(F, 0, 0, torch.device("cuda")), F)
    with disc_path(tc_disc):
        net = TecoGAN(lr, tg, F)
        for _ in range(2):                  # step 1 captures the step graph; later steps replay it
            net.train()
    torch.cuda.synchronize()
    return net


@contextlib.contextmanager
def disc_path(tc_disc):
    """tc_disc False: the dispatch rule of the disblocks turned down for every shape (the fp32 kernels)."""
    fits = K.conv4x4s2_tc_fits
    if not tc_disc:
        K.conv4x4s2_tc_fits = lambda *a: False
    try:
        yield
    finally:
        K.conv4x4s2_tc_fits = fits


def step_ms(net, tc_disc):
    with disc_path(tc_disc):
        t0 = time.perf_counter()
        for _ in range(STEPS):
            net.train()
        torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3 / STEPS


def fp32_conv_share(net):
    from torch.profiler import ProfilerActivity, profile
    with disc_path(False), profile(activities=[ProfilerActivity.CUDA]) as prof:
        net.train()
        torch.cuda.synchronize()
    tot = conv = 0.0
    for e in prof.events():
        if e.device_type == torch.autograd.DeviceType.CUDA:
            us = e.time_range.elapsed_us()
            tot += us
            if "conv2d_f32_kernel" in e.name or "conv2d_wgrad_f32_kernel" in e.name:
                conv += us
    return tot / 1e3, conv / 1e3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--no-step", action="store_true")
    a = ap.parse_args()
    res = {"card": card(), "n": N, "layers": layer_rows()}
    print("card:", res["card"])
    print("%-11s %5s %9s | %-27s | %-27s | %-27s" % ("layer", "out", "Cin>Cout", "fwd us fp32 / tc (TF/s tc)",
                                                    "dgrad us fp32 / tc (TF/s)", "wgrad us fp32 / tc (TF/s)"))
    for r in res["layers"]:
        print("%-11s %4d² %4d>%-4d | %s | %s | %s" % (r["layer"], r["out"], r["cin"], r["cout"], *[
            "%8.1f / %7.1f (%5.1f)" % (r["fp32_%s_us" % op], r["tc_%s_us" % op], r["tc_%s_tflops" % op])
            for op in ("fwd", "dgrad", "wgrad")]))
    for var in ("fp32", "tc"):
        res["%s_total_us" % var] = sum(r["%s_%s_us" % (var, op)] for r in res["layers"] for op in ("fwd", "dgrad", "wgrad"))
        print("%s: all four layers, forward + both gradients: %.1f us" % (var, res["%s_total_us" % var]))
    if not a.no_step:
        nets = {"fp32": make_net(False), "tc": make_net(True)}
        res["step_ms"] = {k: [] for k in nets}
        for _ in range(3):
            for k, net in nets.items():
                res["step_ms"][k].append(step_ms(net, k == "tc"))
        tot, conv = fp32_conv_share(nets["fp32"])
        res["fp32_disc_step_profile_ms"] = {"all_kernels": tot, "conv2d_f32_and_wgrad": conv}
        for k, v in res["step_ms"].items():
            print("bf16 TecoGAN step, disblocks on %s: %s ms/step" % (k, " ".join("%.2f" % t for t in v)))
        print("profiled step with fp32 disblocks: %.2f ms of kernels, %.2f ms (%.1f %%) in conv2d_f32 / conv2d_wgrad_f32"
              % (tot, conv, 100.0 * conv / tot))
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "ab_disc.json"), "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
