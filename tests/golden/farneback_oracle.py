"""Host restatement of cv2.calcOpticalFlowFarneback(prev, next, None, 0.5, 3, 15, 3, 5, 1.2, 0) -- the flow behind the
reference's tOF (metrics.py:143-169) -- written stage by stage in numpy from Farneback (2003) and from black-box probes of
cv2 4.13 (DESIGN.md section 4.4).  Test infrastructure only: product code never imports it.  make_golden_tof.py checks it
against cv2's own flows; tests/test_gpu_tof.py uses each stage as the reference of the matching CUDA kernel.

Arrays are float32 wherever cv2 keeps a float Mat (blurred level, polynomial coefficients, the per-pixel matrix field,
the flow) and float64 where cv2 sums in double (the horizontal polynomial pass, the box filter and the 2x2 solve).
Every float32 expression is evaluated one rounded operation at a time, in the order of the CUDA kernels.
"""
import numpy as np

f32, f64 = np.float32, np.float64

PYR_SCALE, LEVELS, WINSIZE, ITERATIONS, POLY_N, POLY_SIGMA = 0.5, 3, 15, 3, 5, 1.2
MIN_SIZE = 32                                   # a level whose width or height would fall below this is dropped
BORDER = np.array([0.14, 0.14, 0.4472, 0.4472, 0.4472], f32)   # weights of the 5 outermost rows / columns


def grey(rgb_u8):
    """cv2.cvtColor(rgb, COLOR_RGB2GRAY) on uint8: (9798 R + 19235 G + 3735 B + 16384) >> 15, bit for bit."""
    a = np.asarray(rgb_u8).astype(np.int64)
    return ((9798 * a[..., 0] + 19235 * a[..., 1] + 3735 * a[..., 2] + 16384) >> 15).astype(np.uint8)


def num_levels(h, w):
    """Pyramid levels above the full-resolution one: a level is kept while both sides scaled stay >= 32."""
    k, scale = 0, 1.0
    while k < LEVELS:
        scale *= PYR_SCALE
        if w * scale < MIN_SIZE or h * scale < MIN_SIZE:
            break
        k += 1
    return k


def level_size(h, w, k):
    """(height, width) of level k: round-half-to-even of the scaled full size."""
    scale = PYR_SCALE ** k
    return int(round(h * scale)), int(round(w * scale))


def blur_params(k):
    """(sigma, ksize) of the Gaussian applied to the full-resolution image before it is resized to level k."""
    scale = PYR_SCALE ** k
    sigma = (1.0 / scale - 1.0) * 0.5
    ksize = max(int(round(sigma * 5)) | 1, 3)
    return sigma, ksize


def gauss_kernel(ksize, sigma):
    """cv2.getGaussianKernel as float32; sigma <= 0 with ksize 3 is the fixed (1/4, 1/2, 1/4)."""
    if sigma <= 0:
        assert ksize == 3
        return np.array([0.25, 0.5, 0.25], f32)
    x = np.arange(ksize, dtype=f64) - (ksize - 1) / 2
    g = np.exp(-x * x / (2 * sigma * sigma))
    return (g / g.sum()).astype(f32)


def _reflect101(i, n):
    if n == 1:
        return np.zeros_like(i)
    i = np.abs(i)
    return np.where(i >= n, 2 * (n - 1) - i, i)


def _sym_filter(a, kern, axis):
    """Symmetric 1-D filter along `axis` with reflect-101 borders: k0 x0, then += kj (x-j + xj) for j = 1..r."""
    r = len(kern) // 2
    n = a.shape[axis]
    idx = np.arange(n)
    take = lambda off: np.take(a, _reflect101(idx + off, n), axis=axis)   # noqa: E731
    s = (kern[r] * a).astype(f32)
    for j in range(1, r + 1):
        s = (s + f32(kern[r + j]) * (take(-j) + take(j))).astype(f32)
    return s


def _linear_coeffs(src, dst):
    """INTER_LINEAR source index and weight of each destination index (half-pixel centres, edge clamp)."""
    scale = 1.0 / (dst / src)
    f = ((np.arange(dst) + 0.5) * scale - 0.5).astype(f32)
    s = np.floor(f).astype(np.int64)
    f = (f - s.astype(f32)).astype(f32)
    lo = s < 0
    f[lo], s[lo] = 0, 0
    hi = s >= src - 1
    f[hi], s[hi] = 0, src - 1
    return s, np.minimum(s + 1, src - 1), f


def resize_linear(img, oh, ow):
    """cv2.resize(img, (ow, oh), INTER_LINEAR) of a float32 [H,W] or [H,W,C] array; an exact halving in both directions
    is the 2x2 average (cv2 switches to its fast area path there); the same size is a copy."""
    H, W = img.shape[:2]
    if (H, W) == (oh, ow):
        return img.copy()
    if H == 2 * oh and W == 2 * ow:
        a, b, c, d = img[0::2, 0::2], img[0::2, 1::2], img[1::2, 0::2], img[1::2, 1::2]
        return ((((a + b).astype(f32) + c).astype(f32) + d).astype(f32) * f32(0.25)).astype(f32)
    x0, x1, fx = _linear_coeffs(W, ow)
    y0, y1, fy = _linear_coeffs(H, oh)
    ex = (slice(None),) + (None,) * (img.ndim - 2)
    ax, bx = (f32(1) - fx)[ex], fx[ex]
    rows = ((img[:, x0] * ax).astype(f32) + (img[:, x1] * bx).astype(f32)).astype(f32)
    ey = (slice(None), None) + (None,) * (img.ndim - 2)
    ay, by = (f32(1) - fy)[ey], fy[ey]
    return ((rows[y0] * ay).astype(f32) + (rows[y1] * by).astype(f32)).astype(f32)


def pyramid_level(grey_u8, k):
    """Level k of one frame: the FULL-resolution grey image as float32, Gaussian-blurred (reflect-101) with the level's
    sigma / ksize -- level 0 included, with the fixed 3-tap kernel -- then resized INTER_LINEAR to level_size."""
    H, W = grey_u8.shape
    sigma, ksize = blur_params(k)
    kern = gauss_kernel(ksize, sigma)
    b = _sym_filter(_sym_filter(grey_u8.astype(f32), kern, 1), kern, 0)
    return resize_linear(b, *level_size(H, W, k))


def poly_weights():
    """g, x g, x^2 g (float32, taps -5..5) of the normalised Gaussian with sigma 1.2, and the four entries of the inverse
    6x6 moment matrix that turn the weighted sums into coefficients (float64)."""
    n, s = POLY_N, POLY_SIGMA
    x = np.arange(-n, n + 1)
    g = np.exp(-(x * x) / (2 * s * s)).astype(f32)
    g = (g.astype(f64) * (1.0 / g.astype(f64).sum())).astype(f32)
    xg, xxg = (x * g).astype(f32), (x * x * g).astype(f32)
    gd = g.astype(f64)
    G = np.zeros((6, 6))
    for yy in range(-n, n + 1):
        for xx in range(-n, n + 1):
            w = gd[yy + n] * gd[xx + n]
            G[0, 0] += w
            G[1, 1] += w * xx * xx
            G[3, 3] += w * xx ** 4
            G[5, 5] += w * xx * xx * yy * yy
    G[2, 2] = G[0, 3] = G[0, 4] = G[3, 0] = G[4, 0] = G[1, 1]
    G[4, 4] = G[3, 3]
    G[3, 4] = G[4, 3] = G[5, 5]
    iG = np.linalg.inv(G)
    return g, xg, xxg, (iG[1, 1], iG[0, 3], iG[3, 3], iG[5, 5])


def poly_exp(img):
    """Polynomial expansion of a float32 [h,w] level -> [h,w,5] float32 with channels (y, x, yy, xx, xy) coefficients.
    Vertical 11-tap pass in float32 (rows clamped), horizontal 11-tap pass in float64 (columns clamped)."""
    n = POLY_N
    g, xg, xxg, (ig11, ig03, ig33, ig55) = poly_weights()
    h, w = img.shape
    rows = lambda k: img[np.clip(np.arange(h) + k, 0, h - 1)]   # noqa: E731
    v0 = (img * g[n]).astype(f32)
    v1 = np.zeros_like(v0)
    v2 = np.zeros_like(v0)
    for k in range(1, n + 1):
        lo, hi = rows(-k), rows(k)
        p = (lo + hi).astype(f32)
        v0 = (v0 + (g[n + k] * p).astype(f32)).astype(f32)
        v1 = (v1 + (xg[n + k] * (hi - lo).astype(f32)).astype(f32)).astype(f32)
        v2 = (v2 + (xxg[n + k] * p).astype(f32)).astype(f32)
    cols = lambda a, k: a[:, np.clip(np.arange(w) + k, 0, w - 1)].astype(f64)   # noqa: E731
    gd, xgd, xxgd = g.astype(f64), xg.astype(f64), xxg.astype(f64)
    b1, b3, b5 = v0 * gd[n], v1 * gd[n], v2 * gd[n]
    b2, b4, b6 = np.zeros(img.shape), np.zeros(img.shape), np.zeros(img.shape)
    for k in range(1, n + 1):
        l0, r0, l1, r1, l2, r2 = cols(v0, -k), cols(v0, k), cols(v1, -k), cols(v1, k), cols(v2, -k), cols(v2, k)
        b1 += (r0 + l0) * gd[n + k]
        b4 += (r0 + l0) * xxgd[n + k]
        b2 += (r0 - l0) * xgd[n + k]
        b3 += (r1 + l1) * gd[n + k]
        b6 += (r1 - l1) * xgd[n + k]
        b5 += (r2 + l2) * gd[n + k]
    return np.stack([b3 * ig11, b2 * ig11, b1 * ig03 + b5 * ig33, b1 * ig03 + b4 * ig33, b6 * ig55], -1).astype(f32)


def update_matrices(R0, R1, flow):
    """Per-pixel 5-term field (G11, G12, G22, h1, h2) from the two expansions and the current flow: R1 sampled
    bilinearly at x + flow (pixels whose sample square leaves the frame use R0 alone), the border weights on the five
    outermost rows and columns, all in float32, one rounded operation at a time."""
    h, w = flow.shape[:2]
    m = lambda a, b: (a * b).astype(f32)          # noqa: E731
    a_ = lambda a, b: (a + b).astype(f32)         # noqa: E731
    s_ = lambda a, b: (a - b).astype(f32)         # noqa: E731
    dx, dy = flow[..., 0], flow[..., 1]
    X, Y = np.meshgrid(np.arange(w, dtype=f32), np.arange(h, dtype=f32))
    fx, fy = a_(X, dx), a_(Y, dy)
    x1, y1 = np.floor(fx).astype(np.int64), np.floor(fy).astype(np.int64)
    fx, fy = s_(fx, x1.astype(f32)), s_(fy, y1.astype(f32))
    inside = (x1 >= 0) & (x1 < w - 1) & (y1 >= 0) & (y1 < h - 1)
    xc, yc = np.where(inside, x1, 0), np.where(inside, y1, 0)
    one = f32(1)
    a00, a01, a10, a11 = m(s_(one, fx), s_(one, fy)), m(fx, s_(one, fy)), m(s_(one, fx), fy), m(fx, fy)
    r = [a_(a_(a_(m(a00, R1[yc, xc, c]), m(a01, R1[yc, xc + 1, c])), m(a10, R1[yc + 1, xc, c])),
            m(a11, R1[yc + 1, xc + 1, c])) for c in range(5)]
    half, quarter = f32(0.5), f32(0.25)
    r2 = np.where(inside, r[0], f32(0))
    r3 = np.where(inside, r[1], f32(0))
    r4 = np.where(inside, m(a_(R0[..., 2], r[2]), half), R0[..., 2])
    r5 = np.where(inside, m(a_(R0[..., 3], r[3]), half), R0[..., 3])
    r6 = np.where(inside, m(a_(R0[..., 4], r[4]), quarter), m(R0[..., 4], half))
    r2 = m(s_(R0[..., 0], r2), half)
    r3 = m(s_(R0[..., 1], r3), half)
    r2 = a_(r2, a_(m(r4, dy), m(r6, dx)))
    r3 = a_(r3, a_(m(r6, dy), m(r5, dx)))
    edge = lambda i: BORDER[np.minimum(i, 4)]                     # noqa: E731
    xs, ys = np.arange(w), np.arange(h)
    left = np.where(xs < 5, edge(xs), f32(1))[None, :]
    right = np.where(xs >= w - 5, edge(w - 1 - xs), f32(1))[None, :]
    top = np.where(ys < 5, edge(ys), f32(1))[:, None]
    bottom = np.where(ys >= h - 5, edge(h - 1 - ys), f32(1))[:, None]
    scale = m(m(m(left, right), top), bottom)                     # ((left right) top) bottom, as the kernel
    r2, r3, r4, r5, r6 = (m(v, scale) for v in (r2, r3, r4, r5, r6))
    return np.stack([a_(m(r4, r4), m(r6, r6)), m(a_(r4, r5), r6), a_(m(r5, r5), m(r6, r6)),
                     a_(m(r4, r2), m(r6, r3)), a_(m(r6, r2), m(r5, r3))], -1)


def box_solve(M):
    """15x15 box mean of the field (rows and columns clamped, float64) and the regularised 2x2 solve -> flow float32."""
    h, w = M.shape[:2]
    r = WINSIZE // 2
    Md = M.astype(f64)
    v = sum(Md[np.clip(np.arange(h) + k, 0, h - 1)] for k in range(-r, r + 1))
    s = sum(v[:, np.clip(np.arange(w) + k, 0, w - 1)] for k in range(-r, r + 1)) * (1.0 / (WINSIZE * WINSIZE))
    g11, g12, g22, h1, h2 = (s[..., c] for c in range(5))
    idet = 1.0 / (g11 * g22 - g12 * g12 + 1e-3)
    return np.stack([(g11 * h2 - g12 * h1) * idet, (g22 * h1 - g12 * h2) * idet], -1).astype(f32)


def iterate(R0, R1, flow):
    """One update iteration: the matrix field of the current flow, box filter, solve."""
    return box_solve(update_matrices(R0, R1, flow))


def flow_up(flow, h, w):
    """Coarse flow -> next level: INTER_LINEAR resize to (h, w), times 1 / pyr_scale."""
    return (resize_linear(flow, h, w) * f32(1.0 / PYR_SCALE)).astype(f32)


def farneback(prev_u8, next_u8, conditioning=False):
    """The whole flow [H,W,2] float32 of two uint8 grey frames.  conditioning=True also returns the smallest
    eigenvalue of the box-mean 2x2 system of the last full-resolution iteration at each pixel: where it is small the
    system is near-singular, and rounding differences of 1e-7 in its inputs move the flow by far more."""
    H, W = prev_u8.shape
    flow = None
    for k in range(num_levels(H, W), -1, -1):
        h, w = level_size(H, W, k)
        flow = np.zeros((h, w, 2), f32) if flow is None else flow_up(flow, h, w)
        R0, R1 = poly_exp(pyramid_level(prev_u8, k)), poly_exp(pyramid_level(next_u8, k))
        for _ in range(ITERATIONS):
            M = update_matrices(R0, R1, flow)
            flow = box_solve(M)
    if not conditioning:
        return flow
    r = WINSIZE // 2
    Md = M.astype(f64)
    v = sum(Md[np.clip(np.arange(H) + k, 0, H - 1)] for k in range(-r, r + 1))
    s = sum(v[:, np.clip(np.arange(W) + k, 0, W - 1)] for k in range(-r, r + 1)) * (1.0 / (WINSIZE * WINSIZE))
    tr, det = s[..., 0] + s[..., 2], s[..., 0] * s[..., 2] - s[..., 1] ** 2
    return flow, tr / 2 - np.sqrt(np.maximum(tr * tr / 4 - det, 0.0))


def crop_window(h, w):
    """crop_8x8 of the reference (metrics.py:77-92): (y, x, ch, cw)."""
    ch, cw = (h // 32) * 32, (w // 32) * 32
    while ch > h - 16:
        ch -= 32
    while cw > w - 16:
        cw -= 32
    return (h - ch) // 2, (w - cw) // 2, ch, cw


def tof_of_flows(flow_t, flow_o):
    """metrics.py:149-168 on two full-frame flows: crop_8x8, per-pixel L2 norm of the float32 difference, mean (float64)."""
    y, x, ch, cw = crop_window(*flow_t.shape[:2])
    d = np.abs(flow_t[y:y + ch, x:x + cw] - flow_o[y:y + ch, x:x + cw])
    return float(np.sqrt((d * d).sum(-1, dtype=f32)).astype(f64).mean())
