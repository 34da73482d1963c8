"""A/B of the bf16 3x3 convolution (teco_conv3x3_tc) between two builds of libteco.so (TECO_LIB selects the build).

  python tools/ab_conv.py --out DIR                  # run the fixed, seeded case list; DIR/<case>.npy + DIR/times.json
  python tools/ab_conv.py --compare DIR_A DIR_B      # byte-for-byte comparison of two such runs, and their timings

Every case writes its output as raw words (bf16 as 16-bit, fp32 as 32-bit), so --compare checks the results bit for bit.
The list covers the shapes that take the 64 -> 64 one-K-block path: the generator trunk layer at the bench batch (264
clips of 32x32, in-place residual), every activation, ragged images, an image smaller than one tile, fewer tiles than
SMs, a tile count that is not a multiple of the grid, FNet's 64-channel layers and the input-gradient convolution
(flag-3 packing).  It also covers the generator's HR tail at the bench batch, each launch on its own: conv_tran1
(32x32 -> 64x64) and conv_tran2 (64x64 -> 128x128), the fp32 output stage at 128x128 with the bicubic residual, and
FNet's tanh*24 flow head, with ragged and smaller-than-a-tile cases of each.  The output-stage and flow-head cases that
teco_conv3x3_f32out_tc takes run once more on it, as '<case>+f32out' with the same operands; --compare checks those
against the teco_conv3x3_tc case of the same run byte for byte, and across the two runs where both have them."""
import argparse
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

# name: (N, H, W, Cin, Cout, act, residual: None / "inplace" / "separate" / "f32", pack flags, mode, fp32 output channels)
# mode 1 is the 2x transposed convolution (pack flag 1); fp32 output channels c > 0 write [N, H, W, c] fp32 (Cout = 16),
# and "f32" adds an fp32 residual with post = (2, -1): the generator's output stage.
CASES = {
    "trunk_264x32x32_res_inplace": (264, 32, 32, 64, 64, 0, "inplace", 0, 0, 0),
    "trunk_264x32x32_relu": (264, 32, 32, 64, 64, 1, None, 0, 0, 0),
    "lrelu_2x48x40": (2, 48, 40, 64, 64, 2, None, 0, 0, 0),
    "none_2x48x40_res": (2, 48, 40, 64, 64, 0, "separate", 0, 0, 0),
    "ragged_1x19x21_lrelu_res": (1, 19, 21, 64, 64, 2, "separate", 0, 0, 0),
    "ragged_3x19x21_res_inplace": (3, 19, 21, 64, 64, 0, "inplace", 0, 0, 0),
    "small_3x5x6_relu": (3, 5, 6, 64, 64, 1, None, 0, 0, 0),
    "few_tiles_1x128x128_relu": (1, 128, 128, 64, 64, 1, None, 0, 0, 0),
    "odd_tiles_150x32x32_res_inplace": (150, 32, 32, 64, 64, 0, "inplace", 0, 0, 0),   # 1200 tiles on the persistent grid
    "fnet_264x32x32_lrelu": (264, 32, 32, 64, 64, 2, None, 0, 0, 0),
    "fnet_264x16x16_lrelu": (264, 16, 16, 64, 64, 2, None, 0, 0, 0),
    "fnet_264x8x8_to128_lrelu": (264, 8, 8, 64, 128, 2, None, 0, 0, 0),
    "dgrad_flag3_8x32x32": (8, 32, 32, 64, 64, 0, None, 3, 0, 0),
    "vgg_to128_2x64x64_relu": (2, 64, 64, 64, 128, 1, None, 0, 0, 0),
    "wide_cin128_2x32x32_relu": (2, 32, 32, 128, 64, 1, None, 0, 0, 0),                 # two K blocks: the other kernel
    # HR tail
    "tran1_264x32x32_relu": (264, 32, 32, 64, 64, 1, None, 1, 1, 0),
    "tran2_264x64x64_relu": (264, 64, 64, 64, 64, 1, None, 1, 1, 0),
    "tran_ragged_3x19x21_relu": (3, 19, 21, 64, 64, 1, None, 1, 1, 0),
    "tran_small_2x5x6_relu": (2, 5, 6, 64, 64, 1, None, 1, 1, 0),
    "tran_to128_2x24x40_lrelu": (2, 24, 40, 64, 128, 2, None, 1, 1, 0),
    "outstage_264x128x128_bic": (264, 128, 128, 64, 16, 0, "f32", 0, 0, 3),
    "outstage_ragged_3x19x21_bic": (3, 19, 21, 64, 16, 0, "f32", 0, 0, 3),
    "outstage_small_2x5x6_bic": (2, 5, 6, 64, 16, 0, "f32", 0, 0, 3),
    "flowhead_264x32x32_tanh": (264, 32, 32, 64, 16, 3, None, 0, 0, 2),
    "flowhead_ragged_3x19x21_tanh": (3, 19, 21, 64, 16, 3, None, 0, 0, 2),
    "flowhead_small_2x5x6_tanh": (2, 5, 6, 64, 16, 3, None, 0, 0, 2),
}


F32OUT = "+f32out"          # suffix of a case run on teco_conv3x3_f32out_tc


def f32out_cases():
    from tecogan_b200 import kernels as K
    return [n for n, s in CASES.items() if s[9] and K.conv3x3_f32out_fits(s[2], s[9])]


def run_case(name, spec, reps, conv=None):
    from tecogan_b200 import kernels as K
    conv = conv or K.conv3x3_tc
    N, H, W, cin, cout, act, res, flags, mode, f32c = spec
    g = torch.Generator(device="cuda").manual_seed(sum(map(ord, name)))
    x = torch.randn(N, H, W, cin, device="cuda", generator=g).to(torch.bfloat16)
    w = torch.randn(3, 3, cin, cout, device="cuda", generator=g) * (2.0 / (9 * cin)) ** 0.5
    if flags & 1:
        w = w.permute(0, 1, 3, 2).contiguous()
    b = torch.randn(cout, device="cuda", generator=g) * 0.1
    wpk = K.packed_weight(w, cin, cout, flags)
    bias = None if flags == 3 else b
    s = 2 if mode == 1 else 1
    if f32c:
        rf = torch.rand(N, H, W, f32c, device="cuda", generator=g) if res == "f32" else None
        out = torch.empty(N, H, W, f32c, device="cuda")
        post = (2.0, -1.0) if res == "f32" else (1.0, 0.0)

        def launch():
            conv(x, wpk, bias, cout=cout, act=act, out_f32=out, res_f32=rf, post=post)
    else:
        r0 = torch.randn(N, H, W, cout, device="cuda", generator=g).to(torch.bfloat16) if res else None
        out = torch.empty(N, s * H, s * W, cout, device="cuda", dtype=torch.bfloat16)

        def launch():
            if res == "inplace":
                out.copy_(r0)
                K.conv3x3_tc(x, wpk, bias, out, cout=cout, act=act, res=out)
            else:
                K.conv3x3_tc(x, wpk, bias, out, cout=cout, act=act, res=r0, mode=mode)

    launch()
    torch.cuda.synchronize()
    words = out.view(torch.int32 if f32c else torch.int16).cpu().numpy()
    for _ in range(3):
        launch()
    e0, e1, c0, c1 = (torch.cuda.Event(enable_timing=True) for _ in range(4))
    e0.record()
    for _ in range(reps):
        launch()
    e1.record()
    c0.record()                       # the residual copy of the in-place cases, timed alone and subtracted
    for _ in range(reps):
        if res == "inplace":
            out.copy_(r0)
    c1.record()
    torch.cuda.synchronize()
    us = (e0.elapsed_time(e1) - c0.elapsed_time(c1)) * 1000.0 / reps
    return words, us


def work(spec):
    """FLOP the convolution needs and bytes it must move at the least, from the shape: 2 * 9 * Cin * Cout FLOP per input
    pixel, with Cout the real fp32 output channels where there are any (a transposed conv's nine taps are split over its
    four output phases, so it needs no more); the input, the output and the residual moved once each."""
    N, H, W, cin, cout, act, res, flags, mode, f32c = spec
    s = 2 if mode == 1 else 1
    pix = N * H * W
    cout_real = f32c if f32c else cout
    flop = 2.0 * 9 * cin * cout_real * pix
    out_bytes = pix * s * s * (4 * f32c if f32c else 2 * cout)
    res_bytes = pix * (4 * f32c if res == "f32" else (2 * cout if res else 0))
    return flop, pix * cin * 2 + out_bytes + res_bytes


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--out", help="directory for <case>.npy and times.json")
    ap.add_argument("--compare", nargs=2, metavar=("DIR_A", "DIR_B"))
    ap.add_argument("--reps", type=int, default=20)
    args = ap.parse_args()
    if args.compare:
        a, b = args.compare
        ta, tb = (json.load(open(os.path.join(d, "times.json"))) for d in (a, b))
        same = True
        print("%-34s %-10s %10s %10s %9s %9s" % ("case", "outputs", "A us", "B us", "B TFLOP/s", "B GB/s"))
        for name in [n for n in tb if n in ta or n.endswith(F32OUT)]:
            spec = CASES[name[:-len(F32OUT)] if name.endswith(F32OUT) else name]
            xb = np.load(os.path.join(b, name + ".npy"))
            # a '+f32out' case equals the teco_conv3x3_tc case of its own run, and its counterpart in A if A has one
            refs = [os.path.join(b, name[:-len(F32OUT)] + ".npy")] if name.endswith(F32OUT) else []
            refs += [os.path.join(a, name + ".npy")] if name in ta else []
            eq = all(xa.shape == xb.shape and xa.tobytes() == xb.tobytes() for xa in map(np.load, refs))
            same &= eq
            flop, nbytes = work(spec)
            print("%-34s %-10s %10s %10.1f %9.1f %9.0f" % (name, "identical" if eq else "DIFFERENT",
                                                           "%.1f" % ta[name] if name in ta else "-", tb[name],
                                                           flop / tb[name] * 1e-6, nbytes / tb[name] * 1e-3))
        print("all outputs bit-identical" if same else "OUTPUTS DIFFER")
        sys.exit(0 if same else 1)
    if not args.out:
        ap.error("--out DIR or --compare DIR_A DIR_B")
    if not torch.cuda.is_available():
        sys.exit("ab_conv.py needs a GPU")
    os.makedirs(args.out, exist_ok=True)
    times = {}
    for name, spec in CASES.items():
        out, us = run_case(name, spec, args.reps)
        np.save(os.path.join(args.out, name + ".npy"), out)
        times[name] = us
        print("%-34s %9.1f us per launch" % (name, us), flush=True)
    from tecogan_b200 import kernels as K
    for name in f32out_cases():
        out, us = run_case(name, CASES[name], args.reps, K.conv3x3_f32out_tc)
        np.save(os.path.join(args.out, name + F32OUT + ".npy"), out)
        times[name + F32OUT] = us
        print("%-34s %9.1f us per launch" % (name + F32OUT, us), flush=True)
    with open(os.path.join(args.out, "times.json"), "w") as f:
        json.dump(times, f, indent=1)


if __name__ == "__main__":
    main()
