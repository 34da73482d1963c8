"""Functional wrappers over the C ABI (include/teco.h).  Each forward/backward is one or a few of the
hand-written kernels; torch.autograd.Function is used only as the tape that strings them together for
BPTT (plumbing).  All tensors are contiguous NHWC fp32 CUDA tensors unless stated otherwise.
"""
import torch

from . import _ffi as F
from ._ffi import ACT_NONE, ACT_RELU, ACT_LRELU02, ACT_TANH24, ACT_SIGMOID, ConvDesc, TcDesc, call, ptr, stream_ptr

f32 = torch.float32
bf16 = torch.bfloat16


def same_pad(n, k, s):
    """TF 'SAME' padding (before, out) for one axis.  [TF-ext] SURVEY A.2."""
    out = -(-n // s)
    total = max((out - 1) * s + k - n, 0)
    return total // 2, out


def _cc(t):
    return t if t.is_contiguous() else t.contiguous()


# ------------------------------------------------------------------------------------------ raw launches
def conv2d_raw(x, w, bias, y, *, stride, pad_t, pad_l, OH, OW, act=ACT_NONE, res=None, post=(1.0, 0.0),
               out_map=(1, 0, 1, 0), cin=None):
    """One launch of teco_conv2d_f32.  x [N,H,W,Cp] (Cp >= cin channel pitch), w [KH,KW,Cin,Cout] fp32,
    y [N,out_H,out_W,Cout]; out_map = (sy, oy, sx, ox) maps logical output (OH,OW) into y."""
    N, H, W, Cp = x.shape
    KH, KW, Cin, Cout = w.shape
    if cin is None:
        cin = Cp
    if cin != Cin:
        raise ValueError("conv2d: input has %d channels but weights expect %d" % (cin, Cin))
    d = ConvDesc(N=N, H=H, W=W, Cin=Cin, OH=OH, OW=OW, Cout=Cout, KH=KH, KW=KW, stride=stride, pad_t=pad_t, pad_l=pad_l,
                 out_H=y.shape[1], out_W=y.shape[2], out_sy=out_map[0], out_oy=out_map[1], out_sx=out_map[2],
                 out_ox=out_map[3], in_cpitch=Cp, out_cpitch=y.shape[3], act=act, post_scale=post[0], post_shift=post[1])
    call("teco_conv2d_f32", d, ptr(x, f32), ptr(w, f32), ptr(bias, f32), ptr(res, f32), ptr(y, f32), stream_ptr())
    return y


def conv2d_wgrad_raw(x, dy, dw, db, *, stride, pad_t, pad_l, OH, OW, out_map=(1, 0, 1, 0), accumulate=False):
    N, H, W, Cp = x.shape
    KH, KW, Cin, Cout = dw.shape
    d = ConvDesc(N=N, H=H, W=W, Cin=Cin, OH=OH, OW=OW, Cout=Cout, KH=KH, KW=KW, stride=stride, pad_t=pad_t, pad_l=pad_l,
                 out_H=dy.shape[1], out_W=dy.shape[2], out_sy=out_map[0], out_oy=out_map[1], out_sx=out_map[2],
                 out_ox=out_map[3], in_cpitch=Cp, out_cpitch=dy.shape[3], act=0, post_scale=1.0, post_shift=0.0)
    call("teco_conv2d_wgrad_f32", d, ptr(x, f32), ptr(dy, f32), ptr(dw, f32), ptr(db, f32), int(accumulate), stream_ptr())


def _phase_taps(k, pad, a):
    """Transposed-conv phase a (output index i = 2j + a): taps ky with (a + pad - ky) even, ordered by the
    input offset o - j = (a + pad - ky)/2 ascending.  Returns (list of ky, pad_before)."""
    taps = sorted([((a + pad - ky) // 2, ky) for ky in range(k) if (a + pad - ky) % 2 == 0])
    if not taps:
        return [], 0
    offs = [t[0] for t in taps]
    assert offs == list(range(offs[0], offs[0] + len(offs)))
    return [t[1] for t in taps], -offs[0]


def conv_transpose2x_raw(x, w_oi, bias, y, *, pad, act=ACT_NONE):
    """y[n, i, j, co] = sum x[n, o, p, ci] * w_oi[ky, kx, co, ci] with i = 2 o + ky - pad (stride 2), computed as four
    sub-pixel phase convolutions (SURVEY A.3) through the generic conv kernel.  y spatial = 2 * x spatial.
    Used for conv2_tran forward (pad 0) and for the input gradient of stride-2 convs (pad = conv pad)."""
    N, H, W, _ = x.shape
    K = w_oi.shape[0]
    for a in (0, 1):
        kys, pt = _phase_taps(K, pad, a)
        for b in (0, 1):
            kxs, pl = _phase_taps(K, pad, b)
            if not kys or not kxs:
                y[:, a::2, b::2].zero_()
                continue
            # (stack of slices, not list indexing: index tensors would need a host->device copy, which a CUDA graph cannot capture)
            wp = torch.stack([torch.stack([w_oi[ky, kx] for kx in kxs], dim=0) for ky in kys], dim=0)
            wp = wp.permute(0, 1, 3, 2).contiguous()  # [ty,tx,ci,co]
            conv2d_raw(x, wp, bias, y, stride=1, pad_t=pt, pad_l=pl, OH=H, OW=W, act=act, out_map=(2, a, 2, b))
    return y


# ------------------------------------------------------------------------------------------ autograd ops
class _Conv2d(torch.autograd.Function):
    """conv2() = slim.conv2d SAME (+ fused activation, or + residual).  Reference lib/ops.py:47-56."""

    @staticmethod
    def forward(ctx, x, w, b, stride, act, res):
        x, w = _cc(x), _cc(w)
        N, H, W, _ = x.shape
        KH, KW, _, Cout = w.shape
        pt, OH = same_pad(H, KH, stride)
        pl, OW = same_pad(W, KW, stride)
        y = torch.empty((N, OH, OW, Cout), device=x.device, dtype=f32)
        if act != ACT_NONE and res is not None:
            raise ValueError("conv2d: fused activation and residual are mutually exclusive")
        conv2d_raw(x, w, b, y, stride=stride, pad_t=pt, pad_l=pl, OH=OH, OW=OW, act=act, res=None if res is None else _cc(res))
        ctx.cfg = (stride, act, pt, pl, OH, OW, b is not None, res is not None)
        ctx.save_for_backward(x, w, y if act != ACT_NONE else None)
        return y

    @staticmethod
    def backward(ctx, dy):
        stride, act, pt, pl, OH, OW, has_b, has_res = ctx.cfg
        x, w, y = ctx.saved_tensors
        dy = _cc(dy)
        dz = dy
        if act != ACT_NONE:
            dz = torch.empty_like(dy)
            call("teco_act_bwd_f32", ptr(y, f32), ptr(dy, f32), ptr(dz, f32), dy.numel(), act, stream_ptr())
        N, H, W, Cin = x.shape
        KH, KW, _, Cout = w.shape
        dx = dw = db = None
        if ctx.needs_input_grad[0]:
            dx = torch.empty_like(x)
            if stride == 1:
                wf = torch.flip(w, dims=(0, 1)).permute(0, 1, 3, 2).contiguous()  # [kh,kw,Cout,Cin] flipped
                conv2d_raw(dz, wf, None, dx, stride=1, pad_t=KH - 1 - pt, pad_l=KW - 1 - pl, OH=H, OW=W)
            elif stride == 2 and H % 2 == 0 and W % 2 == 0 and pt == pl:
                conv_transpose2x_raw(dz, w, None, dx, pad=pt)   # w is [kh,kw,OUT=Cin,IN=Cout] for this map
            else:
                raise ValueError("conv2d backward: unsupported stride/shape")
        if ctx.needs_input_grad[1]:
            dw = torch.empty_like(w)
            db = torch.empty(Cout, device=x.device, dtype=f32) if has_b and ctx.needs_input_grad[2] else None
            conv2d_wgrad_raw(x, dz, dw, db, stride=stride, pad_t=pt, pad_l=pl, OH=OH, OW=OW)
        return dx, dw, db, None, None, (dy if has_res else None)


def conv2d(x, w, b=None, stride=1, act=ACT_NONE, res=None):
    return _Conv2d.apply(x, w, b, stride, act, res)


class _ConvTranspose2x(torch.autograd.Function):
    """conv2_tran() = slim.conv2d_transpose 3x3 stride 2 SAME.  Reference lib/ops.py:35-44, SURVEY A.3."""

    @staticmethod
    def forward(ctx, x, w, b, act):
        x, w = _cc(x), _cc(w)
        N, H, W, _ = x.shape
        Cout = w.shape[2]
        y = torch.empty((N, 2 * H, 2 * W, Cout), device=x.device, dtype=f32)
        conv_transpose2x_raw(x, w, b, y, pad=0, act=act)
        ctx.act = act
        ctx.has_b = b is not None
        ctx.save_for_backward(x, w, y if act != ACT_NONE else None)
        return y

    @staticmethod
    def backward(ctx, dy):
        x, w, y = ctx.saved_tensors
        dy = _cc(dy)
        dz = dy
        if ctx.act != ACT_NONE:
            dz = torch.empty_like(dy)
            call("teco_act_bwd_f32", ptr(y, f32), ptr(dy, f32), ptr(dz, f32), dy.numel(), ctx.act, stream_ptr())
        N, H, W, Cin = x.shape
        dx = dw = db = None
        if ctx.needs_input_grad[0]:
            dx = torch.empty_like(x)
            # dx[j,ci] = sum_ky dz[2j+ky, co] w[ky,kx,co,ci]: stride-2 conv, pad 0, HWIO = [kh,kw,Cout,Cin] as stored
            conv2d_raw(dz, w, None, dx, stride=2, pad_t=0, pad_l=0, OH=H, OW=W)
        if ctx.needs_input_grad[1]:
            dw = torch.empty_like(w)
            # same conv seen as (input=dz, output grad=x): dW[ky,kx,co,ci]
            conv2d_wgrad_raw(dz, x, dw, None, stride=2, pad_t=0, pad_l=0, OH=H, OW=W)
            if ctx.has_b and ctx.needs_input_grad[2]:
                db = dz.sum(dim=(0, 1, 2))
        return dx, dw, db, None


def conv2d_transpose(x, w, b=None, act=ACT_NONE):
    return _ConvTranspose2x.apply(x, w, b, act)


class _AffineAct(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, a, b, act):
        x = _cc(x)
        y = torch.empty_like(x)
        call("teco_affine_act_f32", ptr(x, f32), ptr(y, f32), x.numel(), a, b, act, stream_ptr())
        ctx.cfg = (a, act)
        ctx.save_for_backward(y if act != ACT_NONE else None)
        return y

    @staticmethod
    def backward(ctx, dy):
        a, act = ctx.cfg
        (y,) = ctx.saved_tensors
        dy = _cc(dy)
        dx = torch.empty_like(dy)
        if act != ACT_NONE:
            call("teco_act_bwd_f32", ptr(y, f32), ptr(dy, f32), ptr(dx, f32), dy.numel(), act, stream_ptr())
            if a != 1.0:
                call("teco_affine_act_f32", ptr(dx, f32), ptr(dx, f32), dx.numel(), a, 0.0, ACT_NONE, stream_ptr())
        else:
            call("teco_affine_act_f32", ptr(dy, f32), ptr(dx, f32), dy.numel(), a, 0.0, ACT_NONE, stream_ptr())
        return dx, None, None, None


def affine_act(x, a=1.0, b=0.0, act=ACT_NONE):
    """y = act(a*x + b): preprocess/deprocess (lib/ops.py:13-22), lrelu (lib/ops.py:84-85), relu, tanh*24, sigmoid."""
    return _AffineAct.apply(x, float(a), float(b), act)


class _MaxPool2(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x):
        x = _cc(x)
        N, H, W, C = x.shape
        y = torch.empty((N, H // 2, W // 2, C), device=x.device, dtype=f32)
        call("teco_maxpool2_f32", ptr(x, f32), ptr(y, f32), N, H, W, C, stream_ptr())
        ctx.save_for_backward(x)
        return y

    @staticmethod
    def backward(ctx, dy):
        (x,) = ctx.saved_tensors
        N, H, W, C = x.shape
        dx = torch.empty_like(x)
        call("teco_maxpool2_bwd_f32", ptr(x, f32), ptr(_cc(dy), f32), ptr(dx, f32), N, H, W, C, stream_ptr())
        return dx


def maxpool2(x):
    return _MaxPool2.apply(x)


class _ResizeBilinear(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, oh, ow):
        x = _cc(x)
        N, h, w, C = x.shape
        y = torch.empty((N, oh, ow, C), device=x.device, dtype=f32)
        call("teco_resize_bilinear_f32", ptr(x, f32), ptr(y, f32), N, h, w, C, oh, ow, stream_ptr())
        ctx.shape = (N, h, w, C, oh, ow)
        return y

    @staticmethod
    def backward(ctx, dy):
        N, h, w, C, oh, ow = ctx.shape
        dx = torch.empty((N, h, w, C), device=dy.device, dtype=f32)
        call("teco_resize_bilinear_bwd_f32", ptr(_cc(dy), f32), ptr(dx, f32), N, h, w, C, oh, ow, stream_ptr())
        return dx, None, None


def resize_bilinear(x, oh, ow):
    """tf.image.resize_images legacy bilinear (lib/frvsr.py:21-22; lib/Teco.py:244; == upscale_four for x4)."""
    return _ResizeBilinear.apply(x, int(oh), int(ow))


class _Warp(torch.autograd.Function):
    @staticmethod
    def forward(ctx, img, flow):
        img, flow = _cc(img), _cc(flow)
        N, H, W, C = img.shape
        if tuple(flow.shape) != (N, H, W, 2):
            raise ValueError("dense_image_warp: flow shape %s does not match image %s" % (tuple(flow.shape), tuple(img.shape)))
        out = torch.empty_like(img)
        call("teco_warp_f32", ptr(img, f32), ptr(flow, f32), ptr(out, f32), N, H, W, C, stream_ptr())
        ctx.save_for_backward(img, flow)
        return out

    @staticmethod
    def backward(ctx, dout):
        img, flow = ctx.saved_tensors
        N, H, W, C = img.shape
        dimg = torch.zeros_like(img) if ctx.needs_input_grad[0] else None
        dflow = torch.empty_like(flow) if ctx.needs_input_grad[1] else None
        call("teco_warp_bwd_f32", ptr(img, f32), ptr(flow, f32), ptr(_cc(dout), f32), ptr(dimg, f32), ptr(dflow, f32),
             N, H, W, C, stream_ptr())
        return dimg, dflow


def dense_image_warp(img, flow):
    """tf.contrib.image.dense_image_warp (lib/Teco.py:120,140,224,254; main.py:215)."""
    return _Warp.apply(img, flow)


class _S2D(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x):
        x = _cc(x)
        N, H, W, C = x.shape
        if H % 4 or W % 4:
            raise ValueError("space_to_depth(4): H and W must be multiples of 4")
        y = torch.empty((N, H // 4, W // 4, 16 * C), device=x.device, dtype=f32)
        call("teco_space_to_depth4_f32", ptr(x, f32), ptr(y, f32), N, H // 4, W // 4, C, 16 * C, 0, stream_ptr())
        ctx.C = C
        return y

    @staticmethod
    def backward(ctx, dy):
        dy = _cc(dy)
        N, h, w, CC = dy.shape
        dx = torch.empty((N, 4 * h, 4 * w, ctx.C), device=dy.device, dtype=f32)
        call("teco_depth_to_space4_f32", ptr(dy, f32), ptr(dx, f32), N, h, w, ctx.C, CC, 0, stream_ptr())
        return dx


def space_to_depth4(x):
    """tf.space_to_depth(x, 4) main.py:201 == lib/Teco.py:145-148."""
    return _S2D.apply(x)


class _BNTrain(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, beta, lrelu):
        x = _cc(x)
        C = x.shape[-1]
        npix = x.numel() // C
        y = torch.empty_like(x)
        stats = torch.empty(4 * C, device=x.device, dtype=f32)
        call("teco_bn_train_f32", ptr(x, f32), ptr(beta, f32), ptr(y, f32), ptr(stats, f32), npix, C, 1e-3, int(lrelu), stream_ptr())
        ctx.lrelu = lrelu
        ctx.save_for_backward(x, y, stats)
        return y

    @staticmethod
    def backward(ctx, dy):
        x, y, stats = ctx.saved_tensors
        C = x.shape[-1]
        npix = x.numel() // C
        dx = torch.empty_like(x)
        dbeta2 = torch.empty(2 * C, device=x.device, dtype=f32)
        call("teco_bn_train_bwd_f32", ptr(x, f32), ptr(y, f32), ptr(_cc(dy), f32), ptr(stats, f32), ptr(dx, f32),
             ptr(dbeta2, f32), npix, C, 1e-3, int(ctx.lrelu), stream_ptr())
        return dx, dbeta2[:C].clone(), None


def batchnorm_train(x, beta, lrelu=False):
    """slim.batch_norm(scale=False, is_training=True, eps=1e-3) (+ fused LeakyReLU 0.2): lib/ops.py:88-90, lib/Teco.py:38-39."""
    return _BNTrain.apply(x, beta, bool(lrelu))


# ------------------------------------------------------------------------------------------ losses (value + fused grad)
class _LossL2(torch.autograd.Function):
    @staticmethod
    def forward(ctx, a, b):
        a, b = _cc(a), _cc(b)
        C = a.shape[-1]
        out = torch.empty(1, device=a.device, dtype=f32)
        da = torch.empty_like(a) if (ctx.needs_input_grad[0] or ctx.needs_input_grad[1]) else None
        call("teco_loss_l2_f32", ptr(a, f32), ptr(b, f32), ptr(out, f32), ptr(da, f32), a.numel() // C, C, 1.0, stream_ptr())
        ctx.save_for_backward(da)
        return out[0]

    @staticmethod
    def backward(ctx, g):
        (da,) = ctx.saved_tensors
        ga = da * g
        return (ga if ctx.needs_input_grad[0] else None), (-ga if ctx.needs_input_grad[1] else None)


def loss_l2(a, b):
    """mean over pixels of sum_c (a-b)^2 -- content / warp loss, lib/Teco.py:320-322, 329-331."""
    return _LossL2.apply(a, b)


class _LossL1(torch.autograd.Function):
    @staticmethod
    def forward(ctx, a, b, per_pixel):
        a, b = _cc(a), _cc(b)
        C = a.shape[-1]
        out = torch.empty(1, device=a.device, dtype=f32)
        da = torch.empty_like(a) if (ctx.needs_input_grad[0] or ctx.needs_input_grad[1]) else None
        call("teco_loss_l1_f32", ptr(a, f32), ptr(b, f32), ptr(out, f32), ptr(da, f32), ptr(None), a.numel() // C, C,
             int(per_pixel), 1.0, stream_ptr())
        ctx.save_for_backward(da)
        return out[0]

    @staticmethod
    def backward(ctx, g):
        (da,) = ctx.saved_tensors
        ga = da * g
        return (ga if ctx.needs_input_grad[0] else None), (-ga if ctx.needs_input_grad[1] else None), None


def loss_l1(a, b, per_pixel=False):
    """mean |a-b| (ping-pong, lib/Teco.py:364-367) or mean over pixels of sum_c |a-b| (D layer loss, :295-296)."""
    return _LossL1.apply(a, b, per_pixel)


class _LossCos(torch.autograd.Function):
    @staticmethod
    def forward(ctx, f, g):
        f, g = _cc(f), _cc(g)
        C = f.shape[-1]
        out = torch.empty(1, device=f.device, dtype=f32)
        df = torch.empty_like(f) if ctx.needs_input_grad[0] else None
        call("teco_loss_cosine_f32", ptr(f, f32), ptr(g, f32), ptr(out, f32), ptr(df, f32), f.numel() // C, C, 1.0, stream_ptr())
        ctx.save_for_backward(df)
        return out[0]

    @staticmethod
    def backward(ctx, gr):
        (df,) = ctx.saved_tensors
        return (df * gr if ctx.needs_input_grad[0] else None), None


def loss_cosine(f, g):
    """1 - mean_pixels cos(f, g) on raw VGG features (the per-pixel channel L2 normalisation of
    lib/Teco.py:19-21 folded in), lib/Teco.py:346-349.  Gradient flows to f only (targets are constants)."""
    return _LossCos.apply(f, g)


class _LossGAN(torch.autograd.Function):
    @staticmethod
    def forward(ctx, d_fake, d_real, eps):
        d_fake, d_real = _cc(d_fake), _cc(d_real)
        out = torch.empty(5, device=d_fake.device, dtype=f32)
        g_adv, g_f, g_r = torch.empty_like(d_fake), torch.empty_like(d_fake), torch.empty_like(d_real)
        call("teco_loss_gan_f32", ptr(d_fake, f32), ptr(d_real, f32), ptr(out, f32), ptr(g_adv, f32), ptr(g_f, f32),
             ptr(g_r, f32), d_fake.numel(), eps, 1.0, 1.0, stream_ptr())
        ctx.save_for_backward(g_adv, g_f, g_r)
        return out

    @staticmethod
    def backward(ctx, g):
        g_adv, g_f, g_r = ctx.saved_tensors
        # out[0] = adv (d_fake), out[1] = discrim loss (d_fake, d_real), out[2] = mean log(dr+eps) (d_real),
        # out[3] = mean dr, out[4] = mean df (reported only; no gradient used by the reference)
        n = g_adv.numel()
        dfk = g_adv * g[0] + g_f * g[1]
        drl = g_r * g[1] - g_r * g[2]
        return dfk, drl, None


def loss_gan(d_fake, d_real, eps=1e-12):
    """[t_adversarial_loss, t_discrim_loss, mean log(D_real+eps), mean D_real, mean D_fake] -- lib/Teco.py:376,394-406."""
    return _LossGAN.apply(d_fake, d_real, float(eps))


# ------------------------------------------------------------------------------------------ no-grad helpers
def upscale4(x, scale=1.0):
    N, h, w, C = x.shape
    y = torch.empty((N, 4 * h, 4 * w, C), device=x.device, dtype=f32)
    call("teco_upscale4_f32", ptr(_cc(x), f32), ptr(y, f32), N, h, w, C, float(scale), stream_ptr())
    return y


def bicubic4(x, C=None):
    N, h, w, Cp = x.shape
    C = Cp if C is None else C
    y = torch.empty((N, 4 * h, 4 * w, C), device=x.device, dtype=f32)
    call("teco_bicubic4_f32", ptr(_cc(x), f32), ptr(y, f32), N, h, w, C, Cp, stream_ptr())
    return y


def gauss_down4(hr):
    N, H, W, C = hr.shape
    lr = torch.empty((N, (H - 9) // 4 + 1, (W - 9) // 4 + 1, C), device=hr.device, dtype=f32)
    call("teco_gauss_down4_f32", ptr(_cc(hr), f32), ptr(lr, f32), N, H, W, C, stream_ptr())
    return lr


def to_u8(x01):
    y = torch.empty(x01.shape, device=x01.device, dtype=torch.uint8)
    call("teco_to_u8", ptr(_cc(x01), f32), ptr(y, torch.uint8), x01.numel(), stream_ptr())
    return y


def l2norm_channels(f):
    """f / sqrt(sum_c f^2 + 1e-12) per pixel (VGG19_slim norm_flag, reference lib/Teco.py:19-21); forward only."""
    f = _cc(f.detach())
    y = torch.empty_like(f)
    call("teco_l2norm_channels_f32", ptr(f, f32), ptr(y, f32), f.numel() // f.shape[-1], f.shape[-1], stream_ptr())
    return y


def adam_step(p, m, v, g, lr_t, b1, b2, eps, gscale=1.0):
    call("teco_adam_f32", ptr(p, f32), ptr(m, f32), ptr(v, f32), ptr(g, f32), p.numel(), float(lr_t), float(b1), float(b2),
         float(eps), float(gscale), stream_ptr())


# ------------------------------------------------------------------------------------------ bf16 tensor-core path
def packed_weight(w, cin_pad, cout_pad, transpose_layout=False, cin_perm=None):
    """fp32 TF-layout weights -> K-major SWIZZLE_128B bf16 slab [cin_pad/64][9][cout_pad][64] (device side)."""
    w = _cc(w)
    if int(transpose_layout) & 1:
        cout, cin = w.shape[2], w.shape[3]
    else:
        cin, cout = w.shape[2], w.shape[3]
    out = torch.empty(9 * cin_pad * cout_pad, device=w.device, dtype=bf16)
    perm = None
    if cin_perm is not None:
        perm = torch.tensor(cin_perm, device=w.device, dtype=torch.int32)
        assert perm.numel() == cin_pad
    call("teco_pack_conv3x3_bf16", ptr(w, f32), cin, cout, cin_pad, cout_pad, int(transpose_layout), ptr(perm), ptr(out),
         stream_ptr())
    return out


def pad_bias(b, cout_pad):
    out = torch.zeros(cout_pad, device=b.device, dtype=f32)
    out[: b.numel()] = b
    return out


def conv3x3_tc(x, wpk, bias, y=None, *, cout, act=ACT_NONE, res=None, mode=0, out_f32=None, res_f32=None, post=(1.0, 0.0)):
    """One launch of the wgmma kernel.  x [N,H,W,Cin] bf16; y [N,H(,x2),W(,x2),cout] bf16 (allocated if None and
    out_f32 is None)."""
    N, H, W, Cin = x.shape
    s = 2 if mode == 1 else 1
    if y is None and out_f32 is None:
        y = torch.empty((N, s * H, s * W, cout), device=x.device, dtype=bf16)
    d = TcDesc(N=N, H=H, W=W, Cin=Cin, Cout=cout, act=act, mode=mode,
               out_f32_c=0 if out_f32 is None else out_f32.shape[-1], post_scale=post[0], post_shift=post[1])
    call("teco_conv3x3_tc", d, ptr(x, bf16), ptr(wpk, bf16), ptr(bias, f32), ptr(res, bf16), ptr(y, bf16), ptr(res_f32, f32),
         ptr(out_f32, f32), stream_ptr())
    return y if out_f32 is None else out_f32


def conv3x3_lin_supported(N, H, W, num_layers):
    from ._ffi import lib
    return bool(lib().teco_conv3x3_lin_supported(N, H, W, num_layers))


def conv3x3_lin_chain(x_in, buf_a, buf_b, wpk_all, bias_all, plan):
    """A chain of 3x3 64->64 layers on 32-pixel-wide images in one launch (teco_conv3x3_lin_tc).  x_in / buf_a / buf_b:
    [N,H,32,64] bf16 (buffer ids 0 / 1 / 2); plan: list of (input id, output id, residual id or -1, activation) per layer;
    wpk_all: the packed layers back to back; bias_all: [L,64] fp32."""
    import ctypes
    N, H, W, C = x_in.shape
    if C != 64:
        raise ValueError("conv3x3_lin_chain: 64-channel NHWC bf16 tensors only (got %d channels)" % C)
    L = len(plan)
    flat = (ctypes.c_int32 * (4 * L))(*[int(v) for row in plan for v in row])
    call("teco_conv3x3_lin_tc", N, H, W, L, ptr(x_in, bf16), ptr(buf_a, bf16), ptr(buf_b, bf16), ptr(wpk_all, bf16),
         ptr(bias_all, f32), ctypes.cast(flat, ctypes.c_void_p), stream_ptr())


def f32_to_bf16_pad(src, dst, C, c_off=0, scale=1.0, shift=0.0):
    npix = src.numel() // src.shape[-1]
    call("teco_f32_to_bf16_pad", ptr(src, f32), ptr(dst, bf16), npix, C, src.shape[-1], dst.shape[-1], c_off, float(scale),
         float(shift), stream_ptr())
    return dst


def bf16_to_f32(src, C=None):
    C = src.shape[-1] if C is None else C
    dst = torch.empty(src.shape[:-1] + (C,), device=src.device, dtype=f32)
    call("teco_bf16_to_f32", ptr(src, bf16), ptr(dst, f32), src.numel() // src.shape[-1], C, src.shape[-1], C, stream_ptr())
    return dst


def maxpool2_bf16(x):
    N, H, W, C = x.shape
    y = torch.empty((N, H // 2, W // 2, C), device=x.device, dtype=bf16)
    call("teco_maxpool2_bf16", ptr(x, bf16), ptr(y, bf16), N, H, W, C, stream_ptr())
    return y


def resize2x_bf16(x):
    N, h, w, C = x.shape
    y = torch.empty((N, 2 * h, 2 * w, C), device=x.device, dtype=bf16)
    call("teco_resize2x_bf16", ptr(x, bf16), ptr(y, bf16), N, h, w, C, stream_ptr())
    return y


def warp_s2d_fused(pre_gen, flow_lr, dst, ch_off, in_scale=1.0, in_shift=0.0, warped_out=None):
    """Fused feedback kernel (teco_warp_s2d_fused): pre_gen [N,4h,4w,3] fp32, flow_lr [N,fh,fw,2] fp32,
    dst [N,h,w,Cp] fp32 or bf16."""
    N, h, w, Cp = dst.shape
    call("teco_warp_s2d_fused", ptr(pre_gen, f32), ptr(flow_lr, f32), ptr(dst), ptr(warped_out, f32), N, h, w,
         flow_lr.shape[1], flow_lr.shape[2], Cp, ch_off, int(dst.dtype == bf16), float(in_scale), float(in_shift), stream_ptr())
    return dst


# ------------------------------------------------------------------------------------------ bf16 tensor-core TRAINING convs
# bf16 compute, fp32 master weights / activations at the autograd boundary (north_star: "bf16 training").  Forward and the
# input gradient run on the wgmma kernel (the input gradient of a 3x3 stride-1 SAME conv is the same conv with the taps
# flipped and Cin/Cout swapped: teco_pack_conv3x3_bf16 flag 3); the weight gradient stays on the fp32 kernel.
_tc_wcache = {}


def tc_cache_clear():
    """Packed bf16 weights are valid for one training step only (call at the start of every step / graph capture)."""
    _tc_wcache.clear()


def _pad64(c):
    return (c + 63) // 64 * 64


def _tc_packed(w, b, flags, cin_pad, cout_pad):
    key = (w.data_ptr(), tuple(w.shape), flags, cin_pad, cout_pad)   # (an address alone can be reused by another weight)
    hit = _tc_wcache.get(key)
    if hit is None:
        wpk = packed_weight(w.detach(), cin_pad, cout_pad, flags)
        bp = None
        if b is not None:
            bp = torch.zeros(cout_pad, device=w.device, dtype=f32)
            bp[: b.numel()].copy_(b.detach())
        hit = _tc_wcache[key] = (wpk, bp)
    return hit


def _to_bf16_rows(x, cpad):
    N, H, W, C = x.shape
    xb = torch.empty((N, H, W, cpad), device=x.device, dtype=bf16)
    call("teco_f32_to_bf16_rowpad", ptr(x, f32), ptr(xb, bf16), N * H * W, C, C, cpad, stream_ptr())
    return xb


def _from_bf16_rows(yb, C, add=None):
    N, H, W, Cp = yb.shape
    y = torch.empty((N, H, W, C), device=yb.device, dtype=f32)
    call("teco_bf16_to_f32_add", ptr(yb, bf16), ptr(add, f32), ptr(y, f32), N * H * W, C, Cp, C, stream_ptr())
    return y


def conv3x3_wgrad_tc(xb, dzb, dw, cin, cout, accumulate=False):
    """dw[3,3,cin,cout] fp32 (+)= sum_p xb[p+tap][ci] dzb[p][co] on wgmma (teco_conv3x3_wgrad_tc); xb / dzb: NHWC bf16 with
    channel counts padded to multiples of 64."""
    N, H, W, cp = xb.shape
    call("teco_conv3x3_wgrad_tc", N, H, W, cp, dzb.shape[-1], cin, cout, ptr(xb, bf16), ptr(dzb, bf16), ptr(dw, f32),
         int(accumulate), stream_ptr())
    return dw


def bias_grad(dz, C=None):
    """db[c] = sum over pixels of dz[..., c] (fp32)."""
    C = dz.shape[-1] if C is None else C
    db = torch.empty(C, device=dz.device, dtype=f32)
    call("teco_bias_grad_f32", ptr(dz, f32), ptr(db, f32), dz.numel() // dz.shape[-1], C, dz.shape[-1], 0, stream_ptr())
    return db


class _Conv3x3TC(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, w, b, act, res):
        x, w = _cc(x), _cc(w)
        if act != ACT_NONE and res is not None:
            raise ValueError("conv2d: fused activation and residual are mutually exclusive")
        Cin, Cout = w.shape[2], w.shape[3]
        cip, cop = _pad64(Cin), _pad64(Cout)
        xb = _to_bf16_rows(x, cip)
        if Cout < 16 and res is None:
            # narrow output (generator 64 -> 3, fnet 32 -> 2): the fp32-output stage of the inference path -- the network's
            # output is not rounded to bf16
            wpk, bp = _tc_packed(w, b, 0, cip, 16)
            y = torch.empty(x.shape[:3] + (Cout,), device=x.device, dtype=f32)
            conv3x3_tc(xb, wpk, bp, None, cout=16, act=act, out_f32=y)
        else:
            wpk, bp = _tc_packed(w, b, 0, cip, cop)
            yb = conv3x3_tc(xb, wpk, bp, cout=cop, act=act)
            y = _from_bf16_rows(yb, Cout, None if res is None else _cc(res))
        ctx.cfg = (act, b is not None, res is not None)
        # the bf16 copy of x feeds the tensor-core weight gradient (half the bytes of the fp32 activation)
        ctx.save_for_backward(xb if ctx.needs_input_grad[1] else None, w, y if act != ACT_NONE else None)
        return y

    @staticmethod
    def backward(ctx, dy):
        act, has_b, has_res = ctx.cfg
        xb, w, y = ctx.saved_tensors
        dy = _cc(dy)
        dz = dy
        if act != ACT_NONE:
            dz = torch.empty_like(dy)
            call("teco_act_bwd_f32", ptr(y, f32), ptr(dy, f32), ptr(dz, f32), dy.numel(), act, stream_ptr())
        Cin, Cout = w.shape[2], w.shape[3]
        cip, cop = _pad64(Cin), _pad64(Cout)
        dx = dw = db = None
        dzb = _to_bf16_rows(dz, cop)
        if ctx.needs_input_grad[0]:
            wpk_t, _ = _tc_packed(w, None, 3, cop, cip)          # flipped taps, Cin <-> Cout
            dxb = conv3x3_tc(dzb, wpk_t, None, cout=cip, act=ACT_NONE)
            dx = _from_bf16_rows(dxb, Cin)
        if ctx.needs_input_grad[1]:
            if Cout % 4 == 0:
                dw = torch.empty_like(w)
                conv3x3_wgrad_tc(xb, dzb, dw, Cin, Cout)          # wgmma, pixels as the contraction dimension
            else:   # 16-byte atomics need Cout % 4 == 0 (generator 64->3, fnet 32->2): dW with Cout rounded up to 4 --
                c4 = (Cout + 3) // 4 * 4                          # the extra columns see the zero pad channels of dzb
                dw4 = torch.empty(w.shape[:3] + (c4,), device=w.device, dtype=f32)
                conv3x3_wgrad_tc(xb, dzb, dw4, Cin, c4)
                dw = dw4[..., :Cout].contiguous()
            if has_b and ctx.needs_input_grad[2]:
                db = bias_grad(dz)
        return dx, dw, db, None, (dy if has_res else None)


def conv3x3_train_tc(x, w, b=None, act=ACT_NONE, res=None):
    return _Conv3x3TC.apply(x, w, b, act, res)


# conv2_tran in bf16 training mode.  y[2j + ky] += x[j] w[ky] (SURVEY A.3), so with dz in space-to-depth form
# dzs[j][(py, px, co)] = dz[2j + py, 2i + px][co] both gradients are ordinary 3x3 stride-1 SAME problems on the LR grid:
#   ky = 0 -> (row offset 0, phase 0), ky = 1 -> (0, 1), ky = 2 -> (+1, 0)          (columns alike)
#   dx[p][ci]  = sum over taps (1+dj, 1+di), c' of dzs[p + (dj, di)][c'] W'[1+dj, 1+di, c', ci]      -> teco_conv3x3_tc
#   dW'[1+dj, 1+di, c', ci] = sum_p dzs[p + (dj, di)][c'] x[p][ci]                                    -> teco_conv3x3_wgrad_tc
# with W'[1+dj(ky), 1+di(kx), (py(ky), px(kx), co), ci] = w[ky, kx, co, ci] and zero elsewhere.
_TCONV_TAP = ((0, 0), (0, 1), (1, 0))         # ky -> (offset, phase)
_tconv_idx = {}


def _tconv_rows():
    """Row of the [36, C, C] view of W' = [ty, tx, phase] that holds w[ky, kx], for the nine (ky, kx) in ky-major order."""
    rows = []
    for ky in range(3):
        for kx in range(3):
            (dj, py), (di, px) = _TCONV_TAP[ky], _TCONV_TAP[kx]
            rows.append(((1 + dj) * 3 + (1 + di)) * 4 + py * 2 + px)
    return rows


def _tconv_index(device):
    """_tconv_rows() as a device tensor (created once per device, outside any CUDA-graph capture: the first step is eager)."""
    t = _tconv_idx.get(device)
    if t is None:
        t = _tconv_idx[device] = torch.tensor(_tconv_rows(), device=device, dtype=torch.int64)
    return t


class _ConvTranspose2xTC(torch.autograd.Function):
    """conv2_tran() 64 -> 64 on wgmma: forward = the 4-phase kernel of the inference path (teco_conv3x3_tc mode 1), input and
    weight gradients through the space-to-depth identities above.  Reference lib/ops.py:35-44 and its TF autodiff."""

    @staticmethod
    def forward(ctx, x, w, b, act):
        x, w = _cc(x), _cc(w)
        Cout, Cin = w.shape[2], w.shape[3]
        wpk, bp = _tc_packed(w, b, 1, Cin, Cout)                  # flag 1: conv_transpose layout [kh,kw,Cout,Cin]
        xb = _to_bf16_rows(x, Cin)
        yb = conv3x3_tc(xb, wpk, bp, cout=Cout, act=act, mode=1)
        y = _from_bf16_rows(yb, Cout)
        ctx.cfg = (act, b is not None)
        ctx.save_for_backward(xb, w, y if act != ACT_NONE else None)
        return y

    @staticmethod
    def backward(ctx, dy):
        act, has_b = ctx.cfg
        xb, w, y = ctx.saved_tensors
        dy = _cc(dy)
        dz = dy
        if act != ACT_NONE:
            dz = torch.empty_like(dy)
            call("teco_act_bwd_f32", ptr(y, f32), ptr(dy, f32), ptr(dz, f32), dy.numel(), act, stream_ptr())
        N, H2, W2, Cout = dz.shape
        H, W, Cin = H2 // 2, W2 // 2, w.shape[3]
        dzb = _to_bf16_rows(dz, Cout)
        dzs = dzb.view(N, H, 2, W, 2, Cout).permute(0, 1, 3, 2, 4, 5).reshape(N, H, W, 4 * Cout)   # one copy: (py, px, co)
        idx = _tconv_index(w.device)
        dx = dw = db = None
        if ctx.needs_input_grad[0]:
            key = (w.data_ptr(), tuple(w.shape), "tconv_dgrad")
            wpk2 = _tc_wcache.get(key)
            if wpk2 is None:
                wp = torch.zeros((36, Cout, Cin), device=w.device, dtype=f32)
                wp.index_copy_(0, idx, w.detach().reshape(9, Cout, Cin))
                wpk2 = _tc_wcache[key] = packed_weight(wp.view(3, 3, 4 * Cout, Cin), 4 * Cout, Cin, 0)
            dxb = conv3x3_tc(dzs, wpk2, None, cout=Cin, act=ACT_NONE)
            dx = _from_bf16_rows(dxb, Cin)
        if ctx.needs_input_grad[1]:
            dwp = torch.empty((3, 3, 4 * Cout, Cin), device=w.device, dtype=f32)
            conv3x3_wgrad_tc(dzs, xb, dwp, 4 * Cout, Cin)        # dzs is the shifted operand, x the unshifted one
            dw = dwp.view(36, Cout, Cin).index_select(0, idx).view(3, 3, Cout, Cin)
            if has_b and ctx.needs_input_grad[2]:
                db = bias_grad(dz)
        return dx, dw, db, None


def conv_transpose2x_train_tc(x, w, b=None, act=ACT_NONE):
    return _ConvTranspose2xTC.apply(x, w, b, act)
