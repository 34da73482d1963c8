"""A/B of the bf16 3x3 convolution (teco_conv3x3_tc) between two builds of libteco.so (TECO_LIB selects the build).

  python tools/ab_conv.py --out DIR                  # run the fixed, seeded case list; DIR/<case>.npy + DIR/times.json
  python tools/ab_conv.py --compare DIR_A DIR_B      # byte-for-byte comparison of two such runs, and their timings

Every case writes its bf16 output as raw 16-bit words, so --compare checks the results bit for bit.  The list covers the
shapes that take the 64 -> 64 one-K-block path: the generator trunk layer at the bench batch (264 clips of 32x32, in-place
residual), every activation, ragged images, an image smaller than one tile, fewer tiles than SMs, a tile count that is
not a multiple of the grid, FNet's 64-channel layers and the input-gradient convolution (flag-3 packing)."""
import argparse
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

# name: (N, H, W, Cin, Cout, act, residual: None / "inplace" / "separate", pack flags)
CASES = {
    "trunk_264x32x32_res_inplace": (264, 32, 32, 64, 64, 0, "inplace", 0),
    "trunk_264x32x32_relu": (264, 32, 32, 64, 64, 1, None, 0),
    "lrelu_2x48x40": (2, 48, 40, 64, 64, 2, None, 0),
    "none_2x48x40_res": (2, 48, 40, 64, 64, 0, "separate", 0),
    "ragged_1x19x21_lrelu_res": (1, 19, 21, 64, 64, 2, "separate", 0),
    "ragged_3x19x21_res_inplace": (3, 19, 21, 64, 64, 0, "inplace", 0),
    "small_3x5x6_relu": (3, 5, 6, 64, 64, 1, None, 0),
    "few_tiles_1x128x128_relu": (1, 128, 128, 64, 64, 1, None, 0),
    "odd_tiles_150x32x32_res_inplace": (150, 32, 32, 64, 64, 0, "inplace", 0),   # 1200 tiles on the persistent grid
    "fnet_264x32x32_lrelu": (264, 32, 32, 64, 64, 2, None, 0),
    "fnet_264x16x16_lrelu": (264, 16, 16, 64, 64, 2, None, 0),
    "fnet_264x8x8_to128_lrelu": (264, 8, 8, 64, 128, 2, None, 0),
    "dgrad_flag3_8x32x32": (8, 32, 32, 64, 64, 0, None, 3),
    "vgg_to128_2x64x64_relu": (2, 64, 64, 64, 128, 1, None, 0),
    "wide_cin128_2x32x32_relu": (2, 32, 32, 128, 64, 1, None, 0),                 # two K blocks: the other kernel
}


def run_case(name, spec, reps):
    from tecogan_b200 import kernels as K
    N, H, W, cin, cout, act, res, flags = spec
    g = torch.Generator(device="cuda").manual_seed(sum(map(ord, name)))
    x = torch.randn(N, H, W, cin, device="cuda", generator=g).to(torch.bfloat16)
    w = torch.randn(3, 3, cin, cout, device="cuda", generator=g) * (2.0 / (9 * cin)) ** 0.5
    if flags & 1:
        w = w.permute(0, 1, 3, 2).contiguous()
    b = torch.randn(cout, device="cuda", generator=g) * 0.1
    wpk = K.packed_weight(w, cin, cout, flags)
    bias = None if flags == 3 else b
    r0 = torch.randn(N, H, W, cout, device="cuda", generator=g).to(torch.bfloat16) if res else None
    y = torch.empty(N, H, W, cout, device="cuda", dtype=torch.bfloat16)

    def launch():
        if res == "inplace":
            y.copy_(r0)
            K.conv3x3_tc(x, wpk, bias, y, cout=cout, act=act, res=y)
        else:
            K.conv3x3_tc(x, wpk, bias, y, cout=cout, act=act, res=r0)

    launch()
    torch.cuda.synchronize()
    out = y.view(torch.int16).cpu().numpy()
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
            y.copy_(r0)
    c1.record()
    torch.cuda.synchronize()
    us = (e0.elapsed_time(e1) - c0.elapsed_time(c1)) * 1000.0 / reps
    return out, us


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
        for name in CASES:
            xa, xb = (np.load(os.path.join(d, name + ".npy")) for d in (a, b))
            eq = xa.shape == xb.shape and xa.tobytes() == xb.tobytes()
            same &= eq
            print("%-34s %s  %9.1f us  %9.1f us" % (name, "identical" if eq else "DIFFERENT", ta[name], tb[name]))
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
    with open(os.path.join(args.out, "times.json"), "w") as f:
        json.dump(times, f, indent=1)


if __name__ == "__main__":
    main()
