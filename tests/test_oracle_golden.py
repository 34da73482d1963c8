"""CPU: the oracle (oracle/teco_oracle.py) against the golden vectors produced by running the
reference's own lib/*.py under the TF shim (tests/golden/make_golden.py).  Pins wiring."""
import ast
import os

import numpy as np
import torch

from oracle import teco_oracle as O
from tests.conftest import GOLDEN

TOL = dict(rtol=2e-5, atol=2e-5)


def _load(name):
    return np.load(os.path.join(GOLDEN, name + ".npz"), allow_pickle=False)


def _t(a):
    return torch.from_numpy(np.asarray(a, dtype=np.float32))


def test_in_tree_resamplers_and_gaussdown():
    g = _load("ops")
    np.testing.assert_allclose(O.bicubic_four(_t(g["x"])).numpy(), g["bicubic_four"], **TOL)
    np.testing.assert_allclose(O.upscale_four(_t(g["f"])).numpy(), g["upscale_four"], **TOL)
    np.testing.assert_allclose(O.gauss_down_by4(_t(g["hr"])).numpy(), g["gauss_down"], **TOL)
    np.testing.assert_allclose(O.deprocess(_t(g["x"])).numpy(), g["deprocess"], **TOL)
    np.testing.assert_allclose(O.preprocess(_t(g["x"])).numpy(), g["preprocess"], **TOL)
    # upscale_four "mimics the tensorflow bilinear-upscaling" (lib/ops.py:126): equals legacy resize
    f = _t(g["f"])
    np.testing.assert_allclose(O.resize_bilinear_legacy(f, f.shape[1] * 4, f.shape[2] * 4).numpy(),
                               g["upscale_four"], **TOL)


def test_generator_matches_reference_wiring():
    for n in (3, 16):
        g = _load("generator_n%d" % n)
        p = O.init_generator(seed=int(g["seed"]), num_resblock=n, bias_std=float(g["bias_std"]))
        out = O.generator_F(p, _t(g["inputs"]), n).numpy()
        np.testing.assert_allclose(out, g["out"], rtol=1e-4, atol=1e-4)


def test_fnet_matches_reference_wiring():
    g = _load("fnet")
    p = O.init_fnet(seed=int(g["seed"]), bias_std=float(g["bias_std"]))
    np.testing.assert_allclose(O.fnet(p, _t(g["inputs"])).numpy(), g["out"], rtol=1e-4, atol=1e-4)


def test_discriminator_matches_reference_wiring():
    g = _load("discriminator")
    p = O.init_discriminator(seed=int(g["seed"]), bias_std=float(g["bias_std"]))
    prob, layers = O.discriminator_F(p, _t(g["inputs"]))
    np.testing.assert_allclose(prob.numpy(), g["prob"], rtol=1e-4, atol=1e-4)
    for i, l in enumerate(layers):
        np.testing.assert_allclose(l.numpy(), g["layer%d" % i], rtol=1e-4, atol=1e-4)


def test_vgg_matches_reference_wiring():
    g = _load("vgg")
    p = O.init_vgg19(seed=int(g["seed"]))
    feats = O.vgg19_features(p, _t(g["inputs"]))
    for i, k in enumerate(O.VGG_TAPS):
        np.testing.assert_allclose(feats[k].numpy(), g["tap%d" % i], rtol=1e-4, atol=1e-5)


def _teco_case(name):
    g = _load(name)
    ci = int(g["ci"])
    fl = ast.literal_eval(str(g["flags"]))
    FL = O.TrainFlags(**fl)
    P = {}
    P.update(O.init_generator(seed=61 + ci, num_resblock=FL.num_resblock, bias_std=0.05))
    P.update(O.init_fnet(seed=71 + ci, bias_std=0.05))
    P.update(O.init_discriminator(seed=81 + ci, bias_std=0.05))
    if FL.vgg_scaling > 0:
        P.update(O.init_vgg19(seed=91 + ci))
    with torch.no_grad():
        res = O.tecogan_forward(P, _t(g["r_inputs"]), _t(g["r_targets"]), FL, bool(g["gan"]))
    assert [str(s) for s in g["update_list_name"]] == res["update_list_name"]
    np.testing.assert_allclose(np.array([float(v) for v in res["update_list"]]), g["update_list"], rtol=2e-4, atol=1e-5)
    T = res["gen_outputs"].shape[1]
    np.testing.assert_allclose(res["gen_outputs"].reshape(-1, *res["gen_outputs"].shape[2:]).numpy(),
                               g["gen_output"], rtol=1e-3, atol=2e-4)
    return T


def test_tecogan_pingpong_losses_match_reference_wiring():
    assert _teco_case("teco_pp") == 5


def test_tecogan_no_pingpong_backward_flow_branch():
    assert _teco_case("teco_nopp") == 4


def test_frvsr_losses_match_reference_wiring():
    assert _teco_case("frvsr") == 3


def test_calendar_fixture_and_warmup_order():
    g = _load("calendar_lr")
    assert g["crop32_u8"].shape == (10, 32, 32, 3) and g["full_u8"].shape == (7, 144, 180, 3)
    assert [str(s) for s in g["order"][:5]] == ["0006.png", "0005.png", "0004.png", "0003.png", "0002.png"]
    assert O.warmup_order(10)[:6] == [5, 4, 3, 2, 1, 0]


def test_conv2d_transpose_is_gradient_of_same_stride2_conv():
    torch.manual_seed(0)
    x, w = torch.randn(2, 5, 7, 4), torch.randn(3, 3, 6, 4)
    inp = torch.zeros(2, 10, 14, 6, requires_grad=True)
    (gr,) = torch.autograd.grad(O.conv2d(inp, w, None, stride=2), inp, x)
    assert (O.conv2d_transpose(x, w) - gr).abs().max().item() < 1e-5


def test_warp_identity_and_integer_shift_and_clamp():
    torch.manual_seed(1)
    im = torch.rand(1, 6, 8, 3)
    z = torch.zeros(1, 6, 8, 2)
    assert torch.equal(O.dense_image_warp(im, z), im)
    fl = z.clone(); fl[..., 0] = 1.0; fl[..., 1] = -2.0     # out[y,x] = im[y-1, x+2], border clamped
    out = O.dense_image_warp(im, fl)
    assert torch.allclose(out[0, 3, 2], im[0, 2, 4]) and torch.allclose(out[0, 0, 7], im[0, 0, 7])


def _warp_clamp_only(image, flow):
    """dense_image_warp's forward value as the oracle computed it before the TF gradient rule: clamp alone."""
    n, h, w, c = image.shape
    qy = torch.arange(h, dtype=image.dtype).view(1, h, 1) - flow[..., 0]
    qx = torch.arange(w, dtype=image.dtype).view(1, 1, w) - flow[..., 1]
    fy, fx = torch.clamp(torch.floor(qy), 0, h - 2), torch.clamp(torch.floor(qx), 0, w - 2)
    ay, ax = torch.clamp(qy - fy, 0.0, 1.0).unsqueeze(-1), torch.clamp(qx - fx, 0.0, 1.0).unsqueeze(-1)
    b, y0, x0 = torch.arange(n).view(n, 1, 1), fy.long(), fx.long()
    tl, tr, bl, br = image[b, y0, x0], image[b, y0, x0 + 1], image[b, y0 + 1, x0], image[b, y0 + 1, x0 + 1]
    top, bot = ax * (tr - tl) + tl, ax * (br - bl) + bl
    return ay * (bot - top) + top


def test_warp_gradient_to_the_flow_follows_tf_at_integer_queries():
    """At zero flow every query is an integer: alpha_raw is 0 everywhere but in row H-1 (y) and column W-1 (x), where
    the floor is clamped to size-2 and alpha_raw is 1.  TF passes the query gradient only where 0 < alpha_raw <= 1, so
    dflow is zero except row H-1 of component 0 and column W-1 of component 1 -- and non-zero there."""
    img, r = _rnd(11, 2, 6, 7, 3), _rnd(12, 2, 6, 7, 3)
    flow = torch.zeros(2, 6, 7, 2, requires_grad=True)
    (d,) = torch.autograd.grad((O.dense_image_warp(img, flow) * r).sum(), flow)
    assert (d[:, :-1, :, 0] == 0).all() and (d[:, :, :-1, 1] == 0).all()
    assert (d[:, -1, :, 0] != 0).all() and (d[:, :, -1, 1] != 0).all()
    # a fractional query keeps its gradient; integer shifts inside the frame have none on that axis
    flow = torch.zeros(2, 6, 7, 2)
    flow[..., 0], flow[..., 1] = 0.25, -1.0
    flow.requires_grad_(True)
    (d,) = torch.autograd.grad((O.dense_image_warp(img, flow) * r).sum(), flow)
    assert (d[:, 1:, :, 0] != 0).all() and (d[:, :, :-2, 1] == 0).all()


def test_warp_forward_value_is_unchanged_by_the_gradient_rule():
    img = _rnd(13, 3, 9, 11, 3)
    for flow in (torch.zeros(3, 9, 11, 2), torch.round(_rnd(14, 3, 9, 11, 2) * 6), _rnd(15, 3, 9, 11, 2) * 4,
                 torch.round(_rnd(16, 3, 9, 11, 2) * 64) / 16, _rnd(17, 3, 9, 11, 2) * 30):
        assert torch.equal(O.dense_image_warp(img, flow), _warp_clamp_only(img, flow))
        assert torch.equal(O.dense_image_warp(img.double(), flow.double()), _warp_clamp_only(img.double(), flow.double()))


def test_inference_sequence_shapes_nonmultiple_of_8():
    pg, pf = O.init_generator(num_resblock=2), O.init_fnet()
    g = _load("calendar_lr")
    frames = [torch.from_numpy(g["full_u8"][i, :44, :36].astype(np.float32) / 255.0) for i in range(3)]
    outs = O.inference_sequence(pg, pf, frames, num_resblock=2)
    assert outs[-1].shape == (176, 144, 3)


def test_tf_adam_matches_closed_form_first_step():
    p = {"a": torch.tensor([1.0, -2.0])}
    opt = O.TFAdam(["a"], p, lr=0.1)
    opt.apply(p, {"a": torch.tensor([0.5, -0.25])})
    # step 1: m=(1-b1)g, v=(1-b2)g^2, lr_t = lr*sqrt(1-b2)/(1-b1) => delta = lr*g/(|g| + eps*sqrt(1-b2)) ~ lr*sign(g)
    assert torch.allclose(p["a"], torch.tensor([0.9, -1.9]), atol=1e-5)


# ---------------------------------------------------------------------------------------------------------------
# [TF-ext] primitives: the oracle's torch restatement against tests/golden/tf_ext_ref.py, a numpy derivation from the
# operators' published definitions that shares no code with the oracle (the goldens above are generated on top of
# tf_ext_ref, so neither check is circular).  Ragged sizes, both strides, clamp cases.
from tests.golden import tf_ext_ref as X  # noqa: E402


def _rnd(seed, *shape, lo=-1.0, hi=1.0):
    g = torch.Generator().manual_seed(seed)
    return torch.rand(*shape, generator=g) * (hi - lo) + lo


def test_tfext_conv2d_same_padding_all_strides():
    for seed, (n, h, w, ci, co, k, s) in enumerate([(2, 7, 9, 5, 4, 3, 1), (1, 8, 8, 3, 6, 3, 2), (2, 9, 7, 4, 3, 4, 2),
                                                    (1, 16, 12, 3, 5, 4, 2), (1, 5, 5, 6, 2, 1, 1), (1, 13, 11, 2, 3, 3, 2)]):
        x, wt, b = _rnd(seed, n, h, w, ci), _rnd(100 + seed, k, k, ci, co), _rnd(200 + seed, co)
        np.testing.assert_allclose(O.conv2d(x, wt, b, s).numpy(), X.conv2d(x.numpy(), wt.numpy(), b.numpy(), s), rtol=1e-5, atol=1e-5)


def test_tfext_conv2d_transpose_is_the_gradient_of_the_same_conv():
    for seed, (n, h, w, ci, co) in enumerate([(1, 4, 5, 3, 2), (2, 7, 3, 4, 5), (1, 1, 1, 2, 2), (1, 6, 6, 8, 8)]):
        x, wt, b = _rnd(seed, n, h, w, ci), _rnd(10 + seed, 3, 3, co, ci), _rnd(20 + seed, co)
        ref = X.conv2d_transpose(x.numpy(), wt.numpy(), b.numpy(), 2)
        assert ref.shape == (n, 2 * h, 2 * w, co)
        np.testing.assert_allclose(O.conv2d_transpose(x, wt, b, 2).numpy(), ref, rtol=1e-5, atol=1e-5)
        # and the definition itself: <conv_T(x), y> == <x, conv_same_s2(y)> with the same filter read as HWIO [kh,kw,Cout->Cin]
        y = _rnd(30 + seed, n, 2 * h, 2 * w, co)
        lhs = float((X.conv2d_transpose(x.numpy(), wt.numpy(), None, 2).astype(np.float64) * y.numpy()).sum())
        rhs = float((x.numpy().astype(np.float64) * X.conv2d(y.numpy(), wt.numpy(), None, 2)).sum())
        assert abs(lhs - rhs) <= 1e-4 * max(1.0, abs(lhs))


def test_tfext_dense_image_warp_axis_order_and_clamp():
    img = _rnd(1, 2, 9, 11, 3)
    # in-range fractional flow, large out-of-range flow (both signs: exercises floor clamp to [0,size-2] and alpha clamp to [0,1])
    for seed, scale in ((2, 1.7), (3, 30.0)):
        flow = _rnd(seed, 2, 9, 11, 2) * scale
        np.testing.assert_allclose(O.dense_image_warp(img, flow).numpy(), X.dense_image_warp(img.numpy(), flow.numpy()),
                                   rtol=1e-5, atol=1e-5)
    # channel 0 of the flow is the ROW displacement: shifting by (+1, 0) reads the pixel one row above
    flow = torch.zeros(2, 9, 11, 2)
    flow[..., 0] = 1.0
    out = X.dense_image_warp(img.numpy(), flow.numpy())
    np.testing.assert_allclose(out[:, 1:], img.numpy()[:, :-1], atol=1e-6)
    np.testing.assert_allclose(O.dense_image_warp(img, flow).numpy(), out, atol=1e-6)


def test_tfext_legacy_resize_batchnorm_pool_s2d():
    x = _rnd(5, 2, 6, 10, 4)
    for oh, ow in ((12, 20), (24, 40), (7, 13), (6, 10)):
        np.testing.assert_allclose(O.resize_bilinear_legacy(x, oh, ow).numpy(), X.resize_bilinear(x.numpy(), oh, ow), rtol=1e-5, atol=1e-6)
    beta = _rnd(6, 4)
    np.testing.assert_allclose(O.batchnorm_train(x, beta, 1e-3).numpy(), X.batch_norm_train(x.numpy(), beta.numpy(), 1e-3), rtol=1e-4, atol=1e-5)
    np.testing.assert_array_equal(O.maxpool(_rnd(7, 1, 7, 9, 3)).numpy(), X.max_pool_2x2(_rnd(7, 1, 7, 9, 3).numpy()))
    y = _rnd(8, 2, 8, 12, 3)
    np.testing.assert_array_equal(O.space_to_depth4(y).numpy(), X.space_to_depth(y.numpy(), 4))
    np.testing.assert_array_equal(O.lrelu(x, 0.2).numpy(), X.leaky_relu(x.numpy(), 0.2))


# ---- evaluation metrics (SURVEY 8f-3): the oracle against the reference's own psnr / crop_8x8 / _rgb2ycbcr outputs
# (tests/golden/make_golden_metrics.py executes those functions out of the reference's metrics.py) --------------------
def _metric_cases():
    g = _load("metrics")
    for i in range(int(g["n_cases"])):
        yield i, g


def test_metrics_psnr_crop_and_y_match_the_reference_functions():
    for i, g in _metric_cases():
        tgt, out = g["tgt%d" % i], g["out%d" % i]
        y, x, h, w = (int(v) for v in g["crop%d" % i])
        ct, co = O.crop_8x8(tgt), O.crop_8x8(out)
        assert ct.shape[:2] == (h, w) and np.array_equal(ct, tgt[y:y + h, x:x + w])
        assert abs(O.psnr_y(tgt, out) - float(g["psnr_full%d" % i])) < 1e-9
        assert abs(O.psnr_y(ct, co) - float(g["psnr_crop%d" % i])) < 1e-9
        if "y_full%d" % i in g.files:
            np.testing.assert_allclose(O._y_of_u8(out), g["y_full%d" % i], rtol=0, atol=1e-10)


def _ssim_direct(tgt, out):
    """Second derivation of compare_ssim's defaults from its definition: explicit 49-term sums per window position,
    sample (co)variances with the 1/(NP-1) normalisation, no filtering library."""
    X, Y = O._y_of_u8(tgt).astype(np.float64), O._y_of_u8(out).astype(np.float64)
    R = Y.max() - Y.min()
    C1, C2 = (0.01 * R) ** 2, (0.03 * R) ** 2
    H, W = X.shape
    tot, n = 0.0, 0
    for r in range(H - 6):
        for c in range(W - 6):
            a, b = X[r:r + 7, c:c + 7].ravel(), Y[r:r + 7, c:c + 7].ravel()
            ua, ub = a.mean(), b.mean()
            va, vb = ((a - ua) ** 2).sum() / 48.0, ((b - ub) ** 2).sum() / 48.0
            vab = ((a - ua) * (b - ub)).sum() / 48.0
            tot += ((2 * ua * ub + C1) * (2 * vab + C2)) / ((ua * ua + ub * ub + C1) * (va + vb + C2))
            n += 1
    return tot / n


def test_metrics_ssim_restatement_equals_the_direct_definition():
    g = _load("metrics")
    tgt, out = g["tgt3"][:40, :37], g["out3"][:40, :37]
    assert abs(O.ssim_y(tgt, out) - _ssim_direct(tgt, out)) < 1e-9
    assert abs(O.ssim_y(tgt, tgt) - 1.0) < 1e-12
    import pytest
    with pytest.raises(ValueError):
        O.ssim_y(tgt[:6], out[:6])
