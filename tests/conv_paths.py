"""Host restatement of how teco_conv3x3_tc, teco_conv3x3_lin_tc and teco_conv3x3_wgrad_tc split a launch into kernels,
Cout slices and tiles (csrc/conv_tc.cu, csrc/conv_wgrad_tc.cu), and of which code paths a launch reaches.

route() mirrors teco_conv3x3_tc, launch_conv3x3 and pick_kernel in conv_tc.cu.  One 64-channel input block, 64-channel
output slices and no fp32 output run on conv3x3_ws_kernel<mode> (72 KB of weights, always resident); any other mode-1
launch is 'refused' (TECO_E_INVALID).  The rest runs on conv3x3_wgmma_kernel<nt>: nt = 64 when Cout % 64 == 0, else 32
when Cout % 32 == 0, else 16, the weights resident when all Cin / 64 blocks fit next to two halo stages (p.resident),
else streamed with each block: <64> is resident for Cin / 64 <= 2, <32> for Cin / 64 <= 4, <16> always.

features() names what one launch reaches: the kernel, its activation, residual kind, Cout, output split, whether the
tile count exceeds the persistent grid, ragged edges, and the epilogue's fp32 features.  tests/test_gpu_conv_exact.py
checks on the host that its case tables reach every required key, and on the GPU that route() names the kernel the
profiler sees.
"""
from collections import namedtuple

SMEM_MAX = 232448                                  # conv_tc.cu SMEM_MAX
HALO_STAGE = 24576                                 # conv_tc.cu HALO_STAGE: 18 x 10 x 128 B rounded up to 1024
TILE_ROWS, TILE_COLS = 16, 8                       # conv_tc.cu TILE_ROWS, TILE_COLS
H100_SMS = 132
# Every conv_tc instance needs at least 50 KB of shared memory (two halo stages), so at most four CTAs fit on an SM and a
# persistent grid has at most 4 x SMs slots (H100 SXM: 132 SMs; fewer SMs only lower the bound).
MAX_SLOTS = 4 * H100_SMS
# conv3x3_trunk_cluster_kernel: clusters of two CTAs, one CTA per SM, so at most SMs / 2 clusters are resident at once
MAX_CLUSTERS = H100_SMS // 2
TR_WSLOTS = 9                                      # conv_tc.cu trunk kernel's weight ring: slot t holds tap t of a layer
WG_ROWS, WG_COLS = 8, 16                           # conv_wgrad_tc.cu WG_ROWS, WG_COLS: weight-gradient tile
ACT_NAMES = ("none", "relu", "lrelu", "tanh24", "sigmoid")

Route = namedtuple("Route", "kernel nt nsplit resident")


def route(mode, cin, cout, res=False, res_is_y=False, out_f32=False, y=True):
    """Kernel instance ('ws<0>', 'wgmma<64>', ..., or 'refused'), output channels per CTA, Cout splits (grid rows) and
    whether the weights are loaded once per CTA.  res_is_y (in-place residual) and y select only tensor maps."""
    del res_is_y, y
    if mode == 1 and (cin != 64 or cout % 64 or res or out_f32):
        return Route("refused", 0, 0, False)
    nblk = cin // 64
    if nblk == 1 and cout % 64 == 0 and not out_f32:
        return Route("ws<%d>" % mode, 64, cout // 64, True)
    nt = 64 if cout % 64 == 0 else (32 if cout % 32 == 0 else 16)
    w_blk_bytes = 9 * nt * 128
    fixed = 1024 + 64 + nt * 4
    resident = fixed + 2 * HALO_STAGE + nblk * w_blk_bytes <= SMEM_MAX
    return Route("wgmma<%d>" % nt, nt, cout // nt, resident)


def tiles(n, h, w):
    return n * -(-h // TILE_ROWS) * -(-w // TILE_COLS)


def features(mode, n, h, w, cin, cout, act, bias=True, res="", y=True, f32c=0, res_f32=False, post=(1.0, 0.0)):
    """Keys '<kernel> <feature>' reached by one teco_conv3x3_tc launch.  res: '' (none), 'sep' or 'inplace'; f32c: the
    fp32 output's channel count (0: no fp32 output)."""
    r = route(mode, cin, cout, bool(res), res == "inplace", f32c > 0, y)
    k = r.kernel
    place = "resident" if r.resident else "streamed"
    out = {k, "%s act=%s" % (k, ACT_NAMES[act]), "%s cout=%d" % (k, cout), "%s cin=%d" % (k, cin), "%s %s" % (k, place),
           "%s res=%s" % (k, res or "none")}
    if res:
        out.add("%s %s+res" % (k, place))
    if not bias:
        out.add("%s bias=None" % k)
    if r.nsplit > 1:
        out.add("%s nsplit>1" % k)
    if tiles(n, h, w) > MAX_SLOTS:
        out.add("%s tiles>grid" % k)
    if h % TILE_ROWS or w % TILE_COLS:
        out.add("%s ragged" % k)
    if h < TILE_ROWS and w < TILE_COLS:
        out.add("%s smaller than a tile" % k)
    if mode == 1 and 0 < h % TILE_ROWS <= TILE_ROWS // 2:
        out.add("%s wg below image" % k)          # the last tile row's lower warpgroup (rows 8..15) has no input row
    if f32c:
        out.add("%s out_f32" % k)
        if cin == 64:
            out.add("%s out_f32 nblk=1" % k)
        if y:
            out.add("%s y+out_f32" % k)
        if f32c > r.nt:
            out.add("%s out_f32_c spans splits" % k)
        if res_f32 and post != (1.0, 0.0) and f32c == 3 and not y:
            out.add("%s output stage" % k)        # the generator's 64 -> 3 (+ bicubic) * 2 - 1
        if ACT_NAMES[act] == "tanh24" and not res_f32 and not y:
            out.add("%s fnet head" % k)           # FNet's 32 -> 2 tanh * 24 flow
    return out


def lin_features(n, h, plan):
    """teco_conv3x3_lin_tc on n 32x32 images (h is 32): conv3x3_trunk_cluster_kernel, one cluster per image at a time
    over a persistent grid of clusters, every layer's nine taps streamed through a TR_WSLOTS-slot weight ring, tap t in
    slot t.  Layer l of a cluster's clip k waits on its slots at parity (k L + l) & 1, so with an even L every clip
    starts on parity 0 and with an odd L the clips alternate."""
    L = len(plan)
    out = {"lin L=%d" % L, "lin last output in buffer %d" % plan[-1][1]}
    if 9 * L > TR_WSLOTS:
        out.add("lin weight ring wraps")          # every slot is refilled for the next layer, at the other parity
    if n > MAX_CLUSTERS:
        out.add("lin clips>clusters")             # a cluster runs several clips: x_in reloaded, partner handshake
    if n > 2 * MAX_CLUSTERS:
        out.add("lin three clips per cluster, L %s" % ("even" if L % 2 == 0 else "odd"))
    for i, o, r, act in plan:
        if r >= 0:
            out.add("lin res=inplace on buffer %d" % r)
        out.add("lin act=%s" % ACT_NAMES[act])
    return out


def wgrad_features(n, h, w, cin, cout):
    out = {"wgrad cout=%d" % cout}
    if h % WG_ROWS or w % WG_COLS:
        out.add("wgrad ragged")
    if cin % 64 or cout % 64:
        out.add("wgrad padded channels")
    if n * -(-h // WG_ROWS) * -(-w // WG_COLS) > 1:
        out.add("wgrad several tiles")                # several atomics into each dw element
    return out
