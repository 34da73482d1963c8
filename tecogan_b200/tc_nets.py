"""bf16 tensor-core execution of generator_F / fnet (reference lib/frvsr.py) on the wgmma kernel.

Activations are NHWC bf16 with channel counts padded to multiples of 64 (one 128-byte swizzled row); weights are re-packed once per
VariableStore version into the K-major SWIZZLE_128B layout (teco_pack_conv3x3_bf16).  The generator input uses an
internal channel order  [0,48) = space-to-depth of the warped previous HR frame, [48,51) = LR RGB, [51,64) = 0
so the fused warp kernel can store 16-byte vectors; the first layer's weights are permuted accordingly.
"""
import ctypes

import torch

from . import kernels as K
from ._ffi import ACT_LRELU02, ACT_NONE, ACT_RELU, ACT_TANH24, call, ptr, stream_ptr
from .variables import current_scope, default_store

bf16 = torch.bfloat16
f32 = torch.float32

GEN_CIN_PERM = [3 + k for k in range(48)] + [0, 1, 2] + [-1] * 13   # packed channel -> reference channel
S2D_OFF, LR_OFF = 0, 48


def pad16(c):
    return (c + 15) // 16 * 16


def pad64(c):
    """bf16 activation tensors carry multiples of 64 channels: 64 ch = one 128-byte swizzled wgmma/TMA row."""
    return (c + 63) // 64 * 64


class TcLayer:
    __slots__ = ("wpk", "bias", "cin_pad", "cout_pad", "cout", "k_live")


def _k_live(live, cin_pad):
    """K-steps of 16 channels per tap that cover `live` input channels of a 64-channel slab (1, 2 or 4); 0 (all) for
    wider inputs."""
    if cin_pad != 64:
        return 0
    return next(k for k in (1, 2, 4) if 16 * k >= live)


_cache = {}


def _layer(full_name, transpose=False, cin_perm=None, cin_pad=None, f32_out=False):
    """Packed weights for variable scope `full_name` (…/Conv or …/Conv2d_transpose), cached per store version."""
    store = default_store()
    key = (store.uid, store.version, full_name)
    L = _cache.get(key)
    if L is not None:
        return L
    w = store[full_name + "/weights"]
    b = store.get(full_name + "/biases")
    if transpose:
        cout, cin = w.shape[2], w.shape[3]
    else:
        cin, cout = w.shape[2], w.shape[3]
    L = TcLayer()
    L.cin_pad = cin_pad or pad64(cin)
    L.cout_pad = pad16(cout) if f32_out else pad64(cout)
    L.cout = cout
    L.k_live = _k_live(cin if cin_perm is None else 1 + max(i for i, c in enumerate(cin_perm) if c >= 0), L.cin_pad)
    L.wpk = K.packed_weight(w.detach(), L.cin_pad, L.cout_pad, transpose, cin_perm)
    L.bias = K.pad_bias(b.detach(), L.cout_pad) if b is not None else None
    for k in [k for k in _cache if k[0] == store.uid and k[2] == full_name]:
        del _cache[k]
    _cache[key] = L
    return L


def _ensure_vars_generator(num_resblock):
    """Create (xavier) any missing generator variable so the tensor-core path can run from a fresh store,
    exactly as the fp32 mirror would on first use."""
    from .variables import get_variable, variable_scope
    def conv(scope, cin, cout, name='Conv', tr=False):
        with variable_scope(scope), variable_scope(name):
            shape = (3, 3, cout, cin) if tr else (3, 3, cin, cout)
            fans = (9 * cout, 9 * cin) if tr else (9 * cin, 9 * cout)
            get_variable('weights', shape, fans=fans)
            get_variable('biases', (cout,), init='zeros')
    with variable_scope('input_stage'):
        conv('conv', 51, 64)
    for i in range(1, num_resblock + 1):
        with variable_scope('resblock_%d' % i):
            conv('conv_1', 64, 64)
            conv('conv_2', 64, 64)
    with variable_scope('conv_tran2highres'):
        conv('conv_tran1', 64, 64, 'Conv2d_transpose', True)
        conv('conv_tran2', 64, 64, 'Conv2d_transpose', True)
    with variable_scope('output_stage'):
        conv('conv', 64, 3)


FNET_SPEC = [("encoder_1", 6, 32), ("encoder_2", 32, 64), ("encoder_3", 64, 128),
             ("decoder_1", 128, 256), ("decoder_2", 256, 128), ("decoder_3", 128, 64)]


def _ensure_vars_fnet():
    from .variables import get_variable, variable_scope
    def conv(scope, cin, cout):
        with variable_scope(scope), variable_scope('Conv'):
            get_variable('weights', (3, 3, cin, cout), fans=(9 * cin, 9 * cout))
            get_variable('biases', (cout,), init='zeros')
    for name, cin, cout in FNET_SPEC:
        with variable_scope(name):
            conv('conv_1', cin, cout)
            conv('conv_2', cout, cout)
    with variable_scope('output_stage'):
        conv('conv1', 64, 32)
        conv('conv2', 32, 2)


# A round of the one-launch trunk takes about as long whether it holds 1 or G clips, while the per-layer launches scale
# with the batch: on an H100 80GB HBM3 (700 W limit) the one launch was 1.35-1.60x faster at 66, 132, 198 and 264 clips
# (full rounds), 1.18x at 33 and 0.83-0.94x at 8 and 67 (1 / 8 and 1 / 2 of a round used); see tools/ab_trunk.py and
# DESIGN 4.1b.  At three and four rounds the two paths cross near a fill of 0.75.
LIN_TRUNK_MIN_FILL = 0.8


class GeneratorPlan:
    """Pre-allocated buffers + packed layers for one (B,h,w) generator shape; `run` issues 2N+5 wgmma launches
    and one bicubic kernel, with no allocation -- safe to capture in a CUDA graph."""

    def __init__(self, scope, B, h, w, num_resblock, device):
        self.B, self.h, self.w, self.nrb = B, h, w, num_resblock
        g = scope + "/"
        self.l_in = _layer(g + "input_stage/conv/Conv", cin_perm=GEN_CIN_PERM, cin_pad=64)
        self.l_res = [(_layer(g + "resblock_%d/conv_1/Conv" % i), _layer(g + "resblock_%d/conv_2/Conv" % i))
                      for i in range(1, num_resblock + 1)]
        self.l_t1 = _layer(g + "conv_tran2highres/conv_tran1/Conv2d_transpose", transpose=True)
        self.l_t2 = _layer(g + "conv_tran2highres/conv_tran2/Conv2d_transpose", transpose=True)
        self.l_out = _layer(g + "output_stage/conv/Conv", f32_out=True)
        z = lambda *s: torch.zeros(s, device=device, dtype=bf16)
        self.x_in = z(B, h, w, 64)            # packed generator input (zero pad channels stay zero)
        self.a = z(B, h, w, 64)
        self.b = z(B, h, w, 64)
        self.u1 = z(B, 2 * h, 2 * w, 64)
        self.u2 = z(B, 4 * h, 4 * w, 64)
        self.bic = torch.zeros((B, 4 * h, 4 * w, 3), device=device, dtype=f32)
        self.out = torch.zeros((B, 4 * h, 4 * w, 3), device=device, dtype=f32)
        self.launches = 2 * num_resblock + 5 + 1
        # the fp32 output stage on its pipelined kernel wherever that takes the shape (any HR width a multiple of 4)
        self.out_conv = K.conv3x3_f32out_tc if K.conv3x3_f32out_fits(4 * w, 3) else K.conv3x3_tc
        # 32x32 frames: the whole trunk can run as one teco_conv3x3_lin_tc launch with the activations in shared memory,
        # taken when the batch fills its rounds of clusters
        # buffer ids: 0 = x_in, 1 = a, 2 = b.  input conv x_in -> a (ReLU); block: a -> b (ReLU), b -> a (+ a)
        plan = [(0, 1, -1, ACT_RELU)] + [(1, 2, -1, ACT_RELU), (2, 1, 1, ACT_NONE)] * num_resblock
        self.lin = False
        if K.conv3x3_lin_in_smem(B, h, w, plan):
            layers = [self.l_in] + [l for pair in self.l_res for l in pair]
            self.trunk_w = torch.cat([l.wpk for l in layers]).contiguous()
            self.trunk_b = torch.cat([l.bias for l in layers]).contiguous()
            self.trunk_plan = plan
            G = K.conv3x3_lin_clusters()
            self.lin = B >= LIN_TRUNK_MIN_FILL * G * -(-B // G)
        if self.lin:
            self.launches = 1 + 4 + 1

    def run_bicubic(self, lr_f32, lr_cpitch=3):
        """bicubic_four(LR) for the output stage (lib/frvsr.py:84-86); independent of everything but the LR frame."""
        call("teco_bicubic4_f32", ptr(lr_f32, f32), ptr(self.bic, f32), self.B, self.h, self.w, 3, lr_cpitch, stream_ptr())

    def run(self, lr_f32, lr_cpitch=3, bicubic=True):
        """x_in must already hold the packed input; lr_f32: fp32 tensor whose first 3 channels are LR RGB
        (bicubic=False: the caller has already issued run_bicubic, e.g. on another stream)."""
        B, h, w = self.B, self.h, self.w
        if bicubic:
            self.run_bicubic(lr_f32, lr_cpitch)
        if self.lin:
            K.conv3x3_lin_chain(self.x_in, self.a, self.b, self.trunk_w, self.trunk_b, self.trunk_plan)
        else:
            K.conv3x3_tc(self.x_in, self.l_in.wpk, self.l_in.bias, self.a, cout=64, act=ACT_RELU)
            for c1, c2 in self.l_res:
                K.conv3x3_tc(self.a, c1.wpk, c1.bias, self.b, cout=64, act=ACT_RELU)
                K.conv3x3_tc(self.b, c2.wpk, c2.bias, self.a, cout=64, act=ACT_NONE, res=self.a)
        K.conv3x3_tc(self.a, self.l_t1.wpk, self.l_t1.bias, self.u1, cout=64, act=ACT_RELU, mode=1)
        K.conv3x3_tc(self.u1, self.l_t2.wpk, self.l_t2.bias, self.u2, cout=64, act=ACT_RELU, mode=1)
        # output stage: conv(64->3) + bicubic_four(LR), then preprocess (*2-1): lib/frvsr.py:79-87
        self.out_conv(self.u2, self.l_out.wpk, self.l_out.bias, None, cout=16, act=ACT_NONE, out_f32=self.out,
                      res_f32=self.bic, post=(2.0, -1.0))
        return self.out


class FNetPlan:
    """Pre-allocated bf16 pipeline for fnet on [n,h,w] inputs: 14 wgmma launches + 3 max-pools + 3 resizes, where an
    encoder's conv_2 runs on the one-K-block warp-specialised kernel (64 input channels, a level of at least 16 x 8) its
    max-pool is fused into the conv's epilogue, and the layers with 6 or 32 live input channels in their 64-channel slab
    (encoder_1, encoder_2/conv_1, the flow head) run only the K-steps that carry them.  t2 of a fused level is not
    written."""

    def __init__(self, scope, n, h, w, device):
        self.n, self.h, self.w = n, h, w
        f = scope + "/"
        self.layers = []
        for name, _, _ in FNET_SPEC:
            self.layers.append((_layer(f + name + "/conv_1/Conv"), _layer(f + name + "/conv_2/Conv")))
        self.l_o1 = _layer(f + "output_stage/conv1/Conv")
        self.l_o2 = _layer(f + "output_stage/conv2/Conv", f32_out=True)
        z = lambda *s: torch.zeros(s, device=device, dtype=bf16)
        self.x_in = z(n, h, w, 64)            # prev RGB (0..2), cur RGB (3..5), zeros
        self.bufs = []
        ch, cw = h, w
        for i, (name, _, cout) in enumerate(FNET_SPEC):
            cp = pad64(cout)
            t1, t2 = z(n, ch, cw, cp), z(n, ch, cw, cp)
            if i < 3:
                ch, cw = ch // 2, cw // 2
            else:
                ch, cw = ch * 2, cw * 2
            self.bufs.append((t1, t2, z(n, ch, cw, cp)))
        self.fh, self.fw = ch, cw
        self.o1 = z(n, ch, cw, 64)
        self.flow = torch.zeros((n, ch, cw, 2), device=device, dtype=f32)
        # levels smaller than conv3x3_tc's 16 x 8 tile of one image run on 128-pixel tiles across images
        self.small = [t2.shape[1] < 16 or t2.shape[2] < 8 for t1, t2, t3 in self.bufs]
        self.fused_pool = [i < 3 and not small and c2.cin_pad == 64
                           for i, ((c1, c2), small) in enumerate(zip(self.layers, self.small))]
        self.launches = 14 + 6 - sum(self.fused_pool)
        self.head_conv = K.conv3x3_f32out_tc if K.conv3x3_f32out_fits(cw, 2) else K.conv3x3_tc

    def run(self, flow_out=None):
        """flow_out: optional fp32 [n,fh,fw,2] destination (default self.flow)."""
        x = self.x_in
        n = self.n
        flow = self.flow if flow_out is None else flow_out
        for i, ((c1, c2), (t1, t2, t3)) in enumerate(zip(self.layers, self.bufs)):
            _, hh, ww, cc = t2.shape
            if self.small[i]:
                K.conv3x3_im2col_tc(x, c1.wpk, c1.bias, t1, cout=c1.cout_pad, act=ACT_LRELU02)
                K.conv3x3_im2col_tc(t1, c2.wpk, c2.bias, t2, cout=c2.cout_pad, act=ACT_LRELU02)
            else:
                K.conv3x3_tc(x, c1.wpk, c1.bias, t1, cout=c1.cout_pad, act=ACT_LRELU02, k_live=c1.k_live)
                K.conv3x3_tc(t1, c2.wpk, c2.bias, t3 if self.fused_pool[i] else t2, cout=c2.cout_pad, act=ACT_LRELU02,
                             k_live=c2.k_live, pool=self.fused_pool[i])
            if i < 3 and not self.fused_pool[i]:
                call("teco_maxpool2_bf16", ptr(t2, bf16), ptr(t3, bf16), n, hh, ww, cc, stream_ptr())
            elif i >= 3:
                call("teco_resize2x_bf16", ptr(t2, bf16), ptr(t3, bf16), n, hh, ww, cc, stream_ptr())
            x = t3
        K.conv3x3_tc(x, self.l_o1.wpk, self.l_o1.bias, self.o1, cout=64, act=ACT_LRELU02, k_live=self.l_o1.k_live)
        self.head_conv(self.o1, self.l_o2.wpk, self.l_o2.bias, None, cout=16, act=ACT_TANH24, out_f32=flow,
                       k_live=self.l_o2.k_live)
        return flow


_plans = {}


def _plan(kind, scope, shape, ctor):
    store = default_store()
    key = (kind, store.uid, store.version, scope) + tuple(shape)
    p = _plans.get(key)
    if p is None:
        for k in [k for k in _plans if k[0] == kind and k[1] == store.uid and k[3] == scope and k[4:] == tuple(shape)]:
            del _plans[k]
        p = _plans[key] = ctor()
    return p


def _f32_slice_to_bf16(src, c_begin, C, dst, c_off):
    """dst[..., c_off:c_off+C] = bf16(src[..., c_begin:c_begin+C]) without materialising the slice."""
    npix = src.numel() // src.shape[-1]
    p = ctypes.c_void_p(src.data_ptr() + 4 * c_begin)
    call("teco_f32_to_bf16_pad", p, ptr(dst, bf16), npix, C, src.shape[-1], dst.shape[-1], c_off, 1.0, 0.0, stream_ptr())


def generator_tc(gen_inputs, gen_output_channels, num_resblock):
    """generator_F on tensor cores for an API-level call (fp32 [B,h,w,51] in, fp32 [B,4h,4w,3] out)."""
    if gen_output_channels != 3:
        raise ValueError("generator_F: gen_output_channels must be 3 (reference main.py:204, lib/Teco.py:88)")
    if gen_inputs.dim() != 4 or gen_inputs.shape[-1] != 51:
        raise ValueError("generator_F: gen_inputs must be [B,h,w,51] (3 LR + 48 space-to-depth channels)")
    gen_inputs = gen_inputs.contiguous()
    B, h, w, _ = gen_inputs.shape
    scope = current_scope()
    _ensure_vars_generator(num_resblock)
    plan = _plan("gen", scope, (B, h, w, num_resblock),
                 lambda: GeneratorPlan(scope, B, h, w, num_resblock, gen_inputs.device))
    _f32_slice_to_bf16(gen_inputs, 3, 48, plan.x_in, S2D_OFF)
    _f32_slice_to_bf16(gen_inputs, 0, 3, plan.x_in, LR_OFF)
    return plan.run(gen_inputs, lr_cpitch=51).clone()


def fnet_tc(fnet_input):
    """fnet on tensor cores for an API-level call (fp32 [n,h,w,6] in, fp32 flow out)."""
    if fnet_input.dim() != 4 or fnet_input.shape[-1] != 6:
        raise ValueError("fnet: fnet_input must be [n,h,w,6]")
    fnet_input = fnet_input.contiguous()
    n, h, w, _ = fnet_input.shape
    if h < 8 or w < 8:
        raise ValueError("fnet: spatial size must be at least 8x8 (three 2x2 max-pools)")
    scope = current_scope()
    _ensure_vars_fnet()
    plan = _plan("fnet", scope, (n, h, w), lambda: FNetPlan(scope, n, h, w, fnet_input.device))
    _f32_slice_to_bf16(fnet_input, 0, 6, plan.x_in, 0)
    return plan.run().clone()
