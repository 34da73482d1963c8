"""Time the 33-layer generator trunk (input conv + 16 residual blocks, 3x3 64->64 on [B,32,32,64] bf16) as one
teco_conv3x3_lin_tc launch against 33 per-layer teco_conv3x3_tc launches, both in CUDA-graph replay, over a sweep of
batches, and check that the two give the same bytes.

    python tools/ab_trunk.py [--batches 8,33,66,...] [--out DIR]

Prints one line per batch and a JSON summary.  With --out, writes each batch's final buffers a and b of the one-launch
path as raw little-endian bf16 words (trunk_B<batch>_{a,b}.bin), so that two builds can be compared byte for byte.
The sweep also runs at G + 1 clips, G being the number of two-CTA clusters resident at once (one more clip than one
round of clusters)."""
import argparse
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from tecogan_b200 import kernels as K  # noqa: E402

L = 33
PLAN = [(0, 1, -1, 1)] + [(1, 2, -1, 1), (2, 1, 1, 0)] * 16
TENSOR_MAC_PER_CLK_SM = 2048          # dense bf16 wgmma, H100 data sheet


def clusters():
    """G: two-CTA clusters resident at once (the one-launch grid is 2 min(B, G) CTAs), from the occupancy query."""
    from tecogan_b200._ffi import lib
    G = lib().teco_conv3x3_lin_clusters()
    assert G > 0, G
    return G


def operands(B, seed=7):
    g = torch.Generator().manual_seed(seed)
    x = (torch.rand(B, 32, 32, 64, generator=g) * 2 - 1).to(torch.bfloat16).cuda()
    ws = [(torch.rand(3, 3, 64, 64, generator=g) * 2 - 1) * (3.0 / 576) ** 0.5 for _ in range(L)]
    bs = [(torch.rand(64, generator=g) - 0.5) * 0.1 for _ in range(L)]
    wpk = [K.packed_weight(w.cuda(), 64, 64) for w in ws]
    return x, wpk, [b.cuda() for b in bs]


def graph_ms(fn, replays=20):
    fn()
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        fn()
    g.replay()
    torch.cuda.synchronize()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(replays):
        g.replay()
    e.record()
    e.synchronize()
    return s.elapsed_time(e) / replays


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", default="8,33,66,132,198,264")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "ab_trunk.py needs a GPU"
    batches = [int(v) for v in args.batches.split(",")]
    G = clusters()
    if G + 1 not in batches:
        batches.append(G + 1)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
    rows = []
    for B in sorted(batches):
        x, wpk, bias = operands(B)
        wall, ball = torch.cat(wpk).contiguous(), torch.cat(bias).contiguous()
        a1, b1 = torch.zeros_like(x), torch.zeros_like(x)
        a2, b2 = torch.zeros_like(x), torch.zeros_like(x)
        bufs2 = {0: x, 1: a2, 2: b2}

        def one():
            K.conv3x3_lin_chain(x, a1, b1, wall, ball, PLAN)

        def per_layer():
            for l, (i, o, r, act) in enumerate(PLAN):
                K.conv3x3_tc(bufs2[i], wpk[l], bias[l], bufs2[o], cout=64, act=act, res=bufs2[r] if r >= 0 else None)
        t_one = graph_ms(one)
        t_pl = graph_ms(per_layer)
        same = torch.equal(a1.view(torch.int16), a2.view(torch.int16)) and torch.equal(b1.view(torch.int16), b2.view(torch.int16))
        mac = B * 1024 * 576 * 64 * L
        rounds = -(-B // G)
        floor_clk = rounds * 512 * 576 * 64 * L / TENSOR_MAC_PER_CLK_SM   # each SM: half a clip (512 pixels) per round
        row = {"B": B, "one_launch_us": t_one * 1e3, "per_layer_us": t_pl * 1e3, "speedup": t_pl / t_one,
               "bit_identical": same, "rounds": rounds, "mma_floor_clocks_per_sm": floor_clk,
               "one_launch_tflops": 2 * mac / (t_one * 1e-3) / 1e12}
        rows.append(row)
        print("B=%4d  one launch %8.1f us  per-layer %8.1f us  x%.2f  identical=%s" % (B, row["one_launch_us"], row["per_layer_us"],
                                                                                   row["speedup"], same), flush=True)
        if args.out:
            a1.cpu().view(torch.int16).numpy().tofile(os.path.join(args.out, "trunk_B%d_a.bin" % B))
            b1.cpu().view(torch.int16).numpy().tofile(os.path.join(args.out, "trunk_B%d_b.bin" % B))
    print(json.dumps({"gpu": torch.cuda.get_device_name(0), "G": G, "rows": rows}))


if __name__ == "__main__":
    main()
