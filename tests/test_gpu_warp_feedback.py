"""The fused feedback kernels behind teco_warp_s2d_fused -- tf.pad SYMMETRIC + upscale_four(4 flow) + dense_image_warp +
space_to_depth (main.py:201,212-215) -- against the float64 oracle composition, bit for bit, on every path they take per tile,
and teco_deprocess_u8, the other per-frame kernel of the engines' loop, against a float32 restatement.

Why bit equality can be required: with flows on a 2^-6 grid (|4 flow| < 2^10) and pixel values on a 2^-7 grid in [-1, 1] (or
a 2^-8 grid in [0, 1]), every fp32 intermediate of both kernels fits in 24 bits -- the flow upsampling, T + (B - T) dy/4, the
query, floor and clamp, the three bilinear blends, and 0.5 v + 0.5 -- so the fp32 result equals the float64 composition
exactly whatever FMA contraction the compiler chose.  The only rounding left is the final bf16 round-to-nearest-even, which
torch's conversion reproduces.  tests/warp_tiles.py restates on the host which path each tile takes; the CPU test below
keeps the case table honest about the paths it reaches."""
from collections import namedtuple

import numpy as np
import pytest
import torch

from oracle import teco_oracle as O
from tests.warp_tiles import paths

SENTINEL = -3.0          # outside every output range below: [0, 1] or [-1, 1]


def _q6(a):              # 2^-6 grid
    return (np.round(np.asarray(a, np.float64) * 64) / 64).astype(np.float32)


def _bench_field(h, w, phase=0.0):
    """bench.py's smooth motion field (1.5, -0.75) LR px/frame + 0.5 sin / cos waves, phase-shifted per batch element."""
    yy, xx = np.meshgrid(np.linspace(0, 6.28, h), np.linspace(0, 6.28, w), indexing="ij")
    return np.stack((1.5 + 0.5 * np.sin(yy + xx + phase), -0.75 + 0.5 * np.cos(yy - xx + phase)), -1)


def _const(vals, fh, fw):             # one constant flow (LR px) per batch element
    return np.float32(vals)[:, None, None, :] * np.ones((1, fh, fw, 1), np.float32)


def _edges_flows():
    """Constant and piecewise-constant flows (LR px) on an 8 x 64 frame: integer HR queries at -2 .. 0, H-2, H-1, H and far
    outside, and tiles whose bounds meet the interior thresholds with equality -- (-1/4, -1/4): qy_lo = qx_lo = 1 on the
    first tiles; (1/2, 1/2): qy_hi = H-3, qx_hi = W-3 on the last tiles of both kernels."""
    f = _const([(-0.25, -0.25), (0.5, 0.5), (0.0, 0.0), (-20.0, 30.0), (0.0, 0.0)], 8, 64)
    f[4, :4] = (0.0, -0.25)
    f[4, 4:] = (0.5, 0.0)
    return f


# name: N, h, w, flow_lr [N, fh, fw, 2] (seeded rng -> float32 on the 2^-6 grid), pixel range, (in_scale, in_shift), and the
# paths of the case table the case must reach (checked on the host by test_case_table_reaches_every_path_of_both_kernels)
Case = namedtuple("Case", "flows h w lo scale reaches")
CASES = {
    "bench_smooth": Case(lambda r: _q6([_bench_field(256, 256, k) for k in range(2)]), 256, 256, -1.0, (0.5, 0.5),
                         {"v2 full+IY+IX", "v2 full+IY", "v2 full+IX", "v2 full", "v1 smem", "v1 smem+interior"}),
    "bench_rough": Case(lambda r: _q6([_bench_field(256, 256, k) + 3.0 * (r.rand(256, 256, 2) - 0.5) for k in range(2)]),
                        256, 256, -1.0, (0.5, 0.5),
                        {"v2 halves S/S", "v2 halves G/S", "v2 halves G/G", "v1 global", "v1 global+interior"}),
    "metric_config": Case(lambda r: _q6([_bench_field(32, 32, k) for k in range(2)]), 32, 32, -1.0, (0.5, 0.5),
                          {"v2 full+IY", "v1 smem"}),
    "ragged_symmetric_pad": Case(lambda r: _q6([_bench_field(32, 40, k) for k in range(2)]), 37, 45, 0.0, (1.0, 0.0),
                                 {"v2 full+IY+IX", "v2 full+IY", "v2 full+IX", "v2 full", "v1 smem+interior"}),
    "mixed_halves": Case(lambda r: _q6(r.rand(2, 16, 16, 2) * 12 - 6), 16, 16, -1.0, (0.5, 0.5),
                         {"v2 halves S/G", "v2 halves G/S", "v1 global", "v1 smem"}),
    "far_out_of_range": Case(lambda r: _q6(-30 + 40 * (r.rand(2, 48, 70, 2) - 0.5)), 48, 70, -1.0, (0.5, 0.5),
                             {"v2 halves G/G", "v1 global"}),
    "exact_edges": Case(lambda r: _edges_flows(), 8, 64, -1.0, (0.5, 0.5),
                        {"v2 qy_lo==1", "v2 qy_hi==H-3", "v2 qx_lo==1", "v2 qx_hi==W-3",
                         "v1 qy_lo==1", "v1 qy_hi==H-3", "v1 qx_lo==1", "v1 qx_hi==W-3", "v1 smem+interior"}),
    "tiny_3x5": Case(lambda r: _q6(r.rand(2, 2, 3, 2) * 4 - 2), 3, 5, 0.0, (1.0, 0.0), {"v2 full", "v1 smem"}),
    "tiny_1x1": Case(lambda r: _const([(0.0, 0.0), (0.25, -0.25), (-3.0, 5.0)], 1, 1), 1, 1, -1.0, (0.5, 0.5),
                     {"v2 full", "v1 smem"}),
}
REQUIRED = {"v2 full+IY+IX", "v2 full+IY", "v2 full+IX", "v2 full",
            "v2 halves S/S", "v2 halves S/G", "v2 halves G/S", "v2 halves G/G",
            "v1 smem", "v1 smem+interior", "v1 global", "v1 global+interior"}


def _flows(name):
    return CASES[name].flows(np.random.RandomState(sorted(CASES).index(name) + 1))


def test_case_table_reaches_every_path_of_both_kernels():
    """Host classification of every tile of every case (dyadic flows as the GPU test uses them): each case reaches the paths
    it claims, and together they reach all four full-window variants and all four half-tile combinations of v2 and the
    shared-memory / global windows of v1 with and without `interior`."""
    seen = set()
    for name, c in CASES.items():
        f = _flows(name)
        assert f.dtype == np.float32 and np.array_equal(f, _q6(f)) and np.abs(4 * f).max() < 2 ** 10, name
        got = set().union(*(paths(fi, c.h, c.w) for fi in f))
        assert c.reaches <= got, (name, sorted(c.reaches - got))
        seen |= got
    assert REQUIRED <= seen, sorted(REQUIRED - seen)


# ------------------------------------------------------------------------------------------------------------ GPU checks
def _bits(t):
    return t.view(torch.int16) if t.dtype == torch.bfloat16 else t.view(torch.int32)


def _assert_bits(got, exp, what):
    bad = _bits(got) != _bits(exp)
    if bad.any():
        i = tuple(int(v) for v in bad.nonzero()[0])
        raise AssertionError("%s: %d / %d elements differ, first at %s: got %r, expected %r" % (
            what, int(bad.sum()), bad.numel(), i, float(got[i]), float(exp[i])))


def _check_dst(got, exp48, ch_off, what):
    """The 48 channels at ch_off equal exp48 bit for bit; every other channel keeps the sentinel."""
    sent = torch.full((1,), SENTINEL, dtype=got.dtype)
    mine = got[..., ch_off:ch_off + 48]
    unwritten = _bits(mine) == _bits(sent)
    assert not unwritten.any(), "%s: %d of the 48 channels never written" % (what, int(unwritten.sum()))
    _assert_bits(mine, exp48, what)
    rest = torch.cat((got[..., :ch_off], got[..., ch_off + 48:]), -1)
    assert (_bits(rest) == _bits(sent)).all(), "%s: wrote outside channels [%d, %d)" % (what, ch_off, ch_off + 48)


def _run(pre, flow, shape, dtype, ch_off, scale, warped=False):
    from tecogan_b200 import kernels as K
    dst = torch.full(shape, SENTINEL, dtype=dtype, device="cuda")
    wout = torch.full(pre.shape, SENTINEL, device="cuda") if warped else None
    K.warp_s2d_fused(pre, flow, dst, ch_off, in_scale=scale[0], in_shift=scale[1], warped_out=wout)
    torch.cuda.synchronize()
    return dst.cpu(), (wout.cpu() if warped else None)


def _refused(pre, flow, shape, dtype, ch_off, warped=False, dst_elem_off=0):
    """teco_warp_s2d_fused refuses the layout with ValueError and writes nothing.  dst_elem_off: dst starts that many
    elements into its buffer."""
    from tecogan_b200 import kernels as K
    buf = torch.full((int(np.prod(shape)) + dst_elem_off,), SENTINEL, dtype=dtype, device="cuda")
    wout = torch.full(pre.shape, SENTINEL, device="cuda") if warped else None
    with pytest.raises(ValueError, match="teco_warp_s2d_fused: .*(bf16 dst|warped_out)"):
        K.warp_s2d_fused(pre, flow, buf[dst_elem_off:].view(shape), ch_off, warped_out=wout)
    torch.cuda.synchronize()
    sent = torch.full((1,), SENTINEL, dtype=dtype)
    assert (_bits(buf.cpu()) == _bits(sent)).all(), (shape, ch_off, "dst written")
    assert wout is None or (wout == SENTINEL).all(), (shape, ch_off, "warped_out written")


# bf16 layouts (pitch, ch_off): warp_s2d_v2_kernel takes an offset and pitch that are multiples of 8; teco_warp_s2d_fused
# refuses the others.  fp32 destinations, at any offset and with or without warped_out, run warp_s2d_fused_kernel.
BF16_LAYOUTS = ((64, 0), (64, 8), (128, 16))
BF16_REFUSED = ((64, 4), (51, 3), (60, 8))


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(CASES))
def test_warp_s2d_matches_float64_reference_and_refuses_unaligned_bf16(name):
    """Both kernels on the same dyadic inputs: each bf16 layout (v2) equals the bf16 rounding of the float64 composition bit
    for bit, the fp32 destinations and warped_out (v1) equal the float64 values exactly, no channel outside
    [ch_off, ch_off + 48) is touched, and the unaligned bf16 layouts are refused without a write."""
    c = CASES[name]
    flow = _flows(name)
    N, fh, fw, _ = flow.shape
    grid = 2.0 ** (-7 if c.lo < 0 else -8)
    rng = np.random.RandomState(100 + sorted(CASES).index(name))
    img = (c.lo + np.round(rng.rand(N, 4 * c.h, 4 * c.w, 3) * (1 - c.lo) / grid) * grid).astype(np.float32)
    img64 = torch.from_numpy(img).double()
    fl = O.upscale_four(O.pad_symmetric_br(torch.from_numpy(flow).double(), c.h - fh, c.w - fw) * 4.0)
    warped = O.dense_image_warp(img64, fl)
    exp = O.space_to_depth4(warped) * c.scale[0] + c.scale[1]
    assert torch.equal(exp.float().double(), exp) and torch.equal(warped.float().double(), warped)   # exact in fp32
    exp32, exp16 = exp.float(), exp.float().to(torch.bfloat16)

    pre, fl_d = torch.from_numpy(img).cuda(), torch.from_numpy(flow).cuda()
    for pitch, off in BF16_LAYOUTS:
        got, _ = _run(pre, fl_d, (N, c.h, c.w, pitch), torch.bfloat16, off, c.scale)
        _check_dst(got, exp16, off, "%s bf16 pitch %d @%d" % (name, pitch, off))
    for pitch, off in BF16_REFUSED:
        _refused(pre, fl_d, (N, c.h, c.w, pitch), torch.bfloat16, off)
    got, wout = _run(pre, fl_d, (N, c.h, c.w, 48), torch.float32, 0, c.scale, warped=True)
    _check_dst(got, exp32, 0, "%s fp32" % name)
    _assert_bits(wout, warped.float(), "%s warped_out" % name)
    got, _ = _run(pre, fl_d, (N, c.h, c.w, 51), torch.float32, 3, c.scale)
    _check_dst(got, exp32, 3, "%s fp32 pitch 51 @3" % name)


@pytest.mark.gpu
def test_warp_s2d_dispatch_runs_v2_on_bf16_and_v1_on_fp32():
    """The comparisons here compare two kernels: every accepted bf16 layout runs warp_s2d_v2_kernel and every fp32 one
    warp_s2d_fused_kernel.  bf16 with warped_out, at an offset or pitch that is not a multiple of 8, or at an address that
    is not 16-byte aligned raises ValueError and launches nothing."""
    from torch.profiler import ProfilerActivity, profile
    pre = torch.rand(1, 32, 32, 3, device="cuda")
    flow = torch.zeros(1, 8, 8, 2, device="cuda")

    def kernels(fn):
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            fn()
        return [e.key for e in prof.key_averages() if "warp_s2d" in e.key]

    def kernel_run(dtype, pitch, off, warped=False):
        names = kernels(lambda: _run(pre, flow, (1, 8, 8, pitch), dtype, off, (1.0, 0.0), warped))
        assert len(names) == 1, names
        return "v2" if "warp_s2d_v2_kernel" in names[0] else "v1"

    for pitch, off in BF16_LAYOUTS:
        assert kernel_run(torch.bfloat16, pitch, off) == "v2", (pitch, off)
    assert kernel_run(torch.float32, 48, 0) == "v1"
    assert kernel_run(torch.float32, 48, 0, warped=True) == "v1"
    assert kernel_run(torch.float32, 51, 3) == "v1"
    refused = [lambda p=p, o=o: _refused(pre, flow, (1, 8, 8, p), torch.bfloat16, o) for p, o in BF16_REFUSED]
    refused += [lambda: _refused(pre, flow, (1, 8, 8, 64), torch.bfloat16, 0, warped=True),
                lambda: _refused(pre, flow, (1, 8, 8, 64), torch.bfloat16, 0, dst_elem_off=4)]
    for fn in refused:
        assert kernels(fn) == []


@pytest.mark.gpu
@pytest.mark.parametrize("h,rough", [(256, False), (256, True), (32, False), (32, True)])
def test_warp_s2d_v1_and_v2_agree_bit_for_bit_on_continuous_inputs(h, rough):
    """torch.rand frames and the benchmark's un-rounded motion field, smooth and rough.  v1 and v2 evaluate the same
    formulas in the same order, so v2's bf16 output is v1's fp32 output rounded to nearest even, bit for bit.  v2 stays
    within one bf16 ulp of the float64 composition, and v1's fp32 destination and warped_out within the fp32 rounding of
    the query coordinate."""
    N = 2
    g = torch.Generator(device="cuda").manual_seed(h + rough)
    pre = torch.rand(N, 4 * h, 4 * h, 3, device="cuda", generator=g)
    yy, xx = torch.meshgrid(torch.linspace(0, 6.28, h, device="cuda"), torch.linspace(0, 6.28, h, device="cuda"), indexing="ij")
    flow = torch.stack((1.5 + 0.5 * torch.sin(yy + xx), -0.75 + 0.5 * torch.cos(yy - xx)), dim=-1).expand(N, h, h, 2)
    if rough:
        flow = flow + 3.0 * (torch.rand(N, h, h, 2, device="cuda", generator=g) - 0.5)
    flow = flow.contiguous()
    v2, _ = _run(pre, flow, (N, h, h, 64), torch.bfloat16, 0, (0.5, 0.5))
    v1, _ = _run(pre, flow, (N, h, h, 48), torch.float32, 0, (0.5, 0.5))
    f32, wout = _run(pre, flow, (N, h, h, 48), torch.float32, 0, (1.0, 0.0), warped=True)
    _assert_bits(v2[..., :48], v1.to(torch.bfloat16), "v2 vs bf16(v1)")
    assert (_bits(v2[..., 48:]) == _bits(torch.full((1,), SENTINEL, dtype=torch.bfloat16))).all(), "v2 wrote past 48 channels"

    warped = O.dense_image_warp(pre.cpu().double(), O.upscale_four(flow.cpu().double() * 4.0))
    ref = O.space_to_depth4(warped)
    assert (v2[..., :48].double() - (ref * 0.5 + 0.5)).abs().max().item() <= 2.0 ** -8
    # a query near coordinate 4h carries up to half an fp32 ulp of 4h: 2^-18 px at 4h = 128, 2^-15 px at 1024
    tol = 2e-5 * max(1, 4 * h // 128)
    assert (wout.double() - warped).abs().max().item() <= tol
    assert (f32.double() - ref).abs().max().item() <= tol


# ------------------------------------------------------------------------------------------------------- deprocess + uint8
def _deprocess_ref(x):
    """deprocess + save_img (reference lib/ops.py:17-22, 521-523) in float32: y = 0.5 x + 0.5, u8 = trunc(clip(255 y))."""
    y = np.float32(0.5) * x + np.float32(0.5)
    with np.errstate(over="ignore"):          # 255 y overflows to inf for y near the fp32 maximum; clipped to 255
        return y, np.clip(y * np.float32(255), 0, 255).astype(np.uint8)


def _deprocess_inputs():
    """+-1, values beyond +-1 up to the fp32 range, +-0, subnormals, and x = 2 k/255 - 1 with its fp32 neighbours (3 ulps
    each way) for every uint8 boundary k."""
    special = np.float32([1, -1, 0.0, -0.0, 1.5, -1.5, 2, -2, 1e30, -1e30, 3e38, -3e38, 1e-45, -1e-45])
    special = np.concatenate([special, np.nextafter(special[:2], np.float32([2, -2]))])
    b = np.float32(2 * np.arange(256) / 255.0 - 1)
    near = [b]
    up, dn = b, b
    for _ in range(3):
        up, dn = np.nextafter(up, np.float32(np.inf)), np.nextafter(dn, np.float32(-np.inf))
        near += [up, dn]
    return np.concatenate([special] + near).astype(np.float32)


@pytest.mark.gpu
@pytest.mark.parametrize("n", [1, 3, 4, 5, 4 * (2 * 132 * 16 * 256 + 5) + 3])
def test_deprocess_u8_matches_float32_restatement(n):
    """teco_deprocess_u8 with and without the float frame: the scalar tail alone (n < 4), the tail after one vector
    (n = 5), and a size above the grid-stride cap (132 SMs x 16 CTAs x 256 threads x 4 values) with a three-value tail.
    Nothing beyond n is written."""
    from tecogan_b200._ffi import call, ptr, stream_ptr
    vals = _deprocess_inputs()
    if n < len(vals):
        chunks = [vals[s:s + n] for s in range(0, len(vals) - n + 1, n)]      # every value through the tail at n < 4
    else:
        x = np.random.RandomState(n).uniform(-1.25, 1.25, n).astype(np.float32)
        x[:len(vals)] = vals
        x[n // 2:n // 2 + len(vals)] = vals
        x[n - len(vals):] = vals
        chunks = [x]
    for x in chunks:
        y_ref, u_ref = _deprocess_ref(x)
        xd = torch.from_numpy(x).cuda()
        for with_y01 in (True, False):
            y01 = torch.full((n + 8,), SENTINEL, device="cuda")
            y8 = torch.full((n + 8,), 0xA5, dtype=torch.uint8, device="cuda")
            call("teco_deprocess_u8", ptr(xd, torch.float32), ptr(y01[:n] if with_y01 else None, torch.float32),
                 ptr(y8[:n], torch.uint8), n, stream_ptr())
            y01, y8 = y01.cpu().numpy(), y8.cpu().numpy()
            bad = np.nonzero(y8[:n] != u_ref)[0]
            assert bad.size == 0, (with_y01, bad[:4], x[bad[:4]], y8[bad[:4]], u_ref[bad[:4]])
            assert (y8[n:] == 0xA5).all()
            if with_y01:
                assert np.array_equal(y01[:n].view(np.int32), y_ref.view(np.int32))
            assert (y01[n if with_y01 else 0:] == np.float32(SENTINEL)).all()
