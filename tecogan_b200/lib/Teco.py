"""Mirror of the reference's lib/Teco.py: VGG19_slim, discriminator_F, TecoGAN, FRVSR.

The reference builds a TF1 graph once and `sess.run(Net.train)` executes a step.  Here `TecoGAN(...)` returns a
`Network` with the same fields (lib/Teco.py:506-517) where `train` is a callable that runs one full step
(forward over the unrolled recurrence, all losses, gradients, optional D update, G/FNet update) on the batch it
was built with or on a new batch passed as `train(r_inputs, r_targets)`.  All arithmetic is in libteco.so kernels;
torch supplies tensors, views/concats and the autograd tape (BPTT bookkeeping).  Training runs in fp32.
"""
import collections
import math

import torch

from .. import kernels as K
from .._ffi import ACT_LRELU02, ACT_RELU, ACT_SIGMOID
from ..variables import default_store, variable_scope
from .frvsr import fnet, generator_F
from .ops import batchnorm, conv2, denselayer, deprocess, maxpool, upscale_four

VGG_MEAN = [123.68, 116.78, 103.94]  # reference lib/Teco.py:3
VGG_LAYER_LABELS = ['vgg_19/conv2/conv2_2', 'vgg_19/conv3/conv3_4', 'vgg_19/conv4/conv4_4', 'vgg_19/conv5/conv5_4']
_VGG_CFG = [(1, 2, 64), (2, 2, 128), (3, 4, 256), (4, 4, 512), (5, 4, 512)]


_consts = {}


def _const(key, make):
    """Device constants are created once, outside any CUDA-graph capture (host->device copies cannot be captured)."""
    if key not in _consts:
        _consts[key] = make()
    return _consts[key]


def _vgg_raw(input_pm1):
    """vgg_19 conv trunk (reference lib/ops.py:287-334) on deprocess(x)*255 - mean; returns {scope: post-ReLU feature}."""
    x = K.affine_act(input_pm1, 127.5, 127.5)             # deprocess then *255  (lib/Teco.py:9-10)
    mean = _const(("vgg_mean", x.device), lambda: torch.tensor(VGG_MEAN, device=x.device, dtype=torch.float32))
    x = x - mean                                           # per-channel constant shift (plumbing-sized op)
    out = {}
    with variable_scope('vgg_19'):
        for blk, reps, cout in _VGG_CFG:
            with variable_scope('conv%d' % blk):
                for j in range(1, reps + 1):
                    name = 'conv%d_%d' % (blk, j)
                    with variable_scope(name):
                        cin = x.shape[-1]
                        from ..variables import get_variable
                        w = get_variable('weights', (3, 3, cin, cout), fans=(9 * cin, 9 * cout))
                        b = get_variable('biases', (cout,), init='zeros')
                    from .. import config
                    if config.train_precision() == "bf16":
                        x = K.conv3x3_train_tc(x, w, b, ACT_RELU)     # frozen weights: forward (+ input gradient) on wgmma
                    else:
                        x = K.conv2d(x, w, b, 1, ACT_RELU)      # slim.conv2d default activation relu, SAME (lib/Teco.py:12)
                    out['vgg_19/conv%d/%s' % (blk, name)] = x
            if blk < 5:
                x = maxpool(x)
    return out


def VGG19_slim(input, reuse, deep_list=None, norm_flag=True):
    """reference lib/Teco.py:5-24: selected VGG19 feature maps, each divided by its per-pixel channel L2 norm."""
    output = _vgg_raw(input)
    results = {}
    for key in output:
        if (deep_list is None) or (key in deep_list):
            results[key] = K.l2norm_channels(output[key]) if norm_flag else output[key]
    return results


def discriminator_F(dis_inputs, FLAGS=None):
    """reference lib/Teco.py:30-74 -> (sigmoid prob map [tb,h/16,w/16,1], [4 hidden layers])."""
    if FLAGS is None:
        raise ValueError('No FLAGS is provided for generator')

    def discriminator_block(inputs, output_channel, kernel_size, stride, scope):
        with variable_scope(scope):
            net = conv2(inputs, kernel_size, output_channel, stride, use_bias=False, scope='conv1')
            net = batchnorm(net, is_training=True, lrelu02=True)     # BN + lrelu(0.2) fused (lib/Teco.py:38-39)
        return net

    layer_list = []
    with variable_scope('discriminator_unit'):
        with variable_scope('input_stage'):
            net = conv2(dis_inputs, 3, 64, 1, scope='conv', act=ACT_LRELU02)
        for name, cout in (('disblock_1', 64), ('disblock_3', 64), ('disblock_5', 128), ('disblock_7', 256)):
            net = discriminator_block(net, cout, 4, 2, name)
            layer_list += [net]
        with variable_scope('dense_layer_2'):
            net = denselayer(net, 1)
            net = K.affine_act(net, 1.0, 0.0, ACT_SIGMOID)
    return net, layer_list


# ---------------------------------------------------------------------------------------------- training graph
def _flag(FLAGS, name, default):
    return getattr(FLAGS, name, default)


class _Graph:
    """One forward evaluation of the TecoGAN graph (reference lib/Teco.py:77-413) on a batch."""

    def __init__(self, r_inputs, r_targets, FLAGS, GAN_Flag, global_step):
        B, crop, RNN_N = FLAGS.batch_size, FLAGS.crop_size, FLAGS.RNN_N
        if tuple(r_inputs.shape) != (B, RNN_N, crop, crop, 3):
            raise ValueError("TecoGAN: r_inputs must be [batch,RNN_N,crop,crop,3] = %s, got %s"
                             % ((B, RNN_N, crop, crop, 3), tuple(r_inputs.shape)))
        if tuple(r_targets.shape) != (B, RNN_N, 4 * crop, 4 * crop, 3):
            raise ValueError("TecoGAN: r_targets must be [batch,RNN_N,4crop,4crop,3], got %s" % (tuple(r_targets.shape),))
        inputimages = RNN_N
        if FLAGS.pingpang:   # lib/Teco.py:80-85
            r_inputs = torch.cat((r_inputs, torch.flip(r_inputs[:, :-1], dims=(1,))), dim=1)
            r_targets = torch.cat((r_targets, torch.flip(r_targets[:, :-1], dims=(1,))), dim=1)
            inputimages = RNN_N * 2 - 1
        T, H = inputimages, crop * 4
        # ---- fnet on all consecutive pairs (lib/Teco.py:102-117)
        pre, cur = r_inputs[:, :-1], r_inputs[:, 1:]
        fnet_input = torch.cat((pre, cur), dim=-1).reshape(B * (T - 1), crop, crop, 6)
        with variable_scope('fnet'):
            gen_flow_lr = fnet(fnet_input, reuse=False)
        gen_flow = upscale_four(K.affine_act(gen_flow_lr, 4.0, 0.0)).reshape(B, T - 1, H, H, 2)
        input_frames = cur.reshape(B * (T - 1), crop, crop, 3)
        s_input_warp = K.dense_image_warp(pre.reshape(B * (T - 1), crop, crop, 3).contiguous(), gen_flow_lr)  # :120-122
        # ---- recurrent generator (lib/Teco.py:125-164)
        zeros48 = torch.zeros((B, crop, crop, 48), device=r_inputs.device, dtype=torch.float32)
        gen_outputs, gen_warppre = [], []
        with variable_scope('generator'):
            gen_pre = generator_F(torch.cat((r_inputs[:, 0], zeros48), dim=-1), 3, reuse=False, FLAGS=FLAGS)
            gen_outputs.append(gen_pre)
            for t in range(T - 1):
                warped = K.dense_image_warp(gen_pre, gen_flow[:, t].contiguous())
                gen_warppre.append(warped)
                s2d = K.space_to_depth4(deprocess(warped))
                gen_pre = generator_F(torch.cat((r_inputs[:, t + 1], s2d), dim=-1), 3, reuse=True, FLAGS=FLAGS)
                gen_outputs.append(gen_pre)
        gen_outputs = torch.stack(gen_outputs, dim=1)
        s_gen_output = gen_outputs.reshape(B * T, H, H, 3)
        s_targets = r_targets.reshape(B * T, H, H, 3)

        update_list, update_list_name = [], []
        vgg_on = FLAGS.vgg_scaling > 0.0
        if vgg_on:   # :174-178 -- raw features; the channel normalisation is folded into the cosine loss kernel
            gen_vgg = _vgg_raw(s_gen_output)
            with torch.no_grad():
                target_vgg = _vgg_raw(s_targets)

        dt_ratio = min(FLAGS.Dt_ratio_max, FLAGS.Dt_ratio_0 + FLAGS.Dt_ratio_add * float(global_step))
        if GAN_Flag:  # :180-313
            if not FLAGS.Dt_mergeDs:
                # The reference's own non-merged branch cannot run either: lib/Teco.py:248,269 bind the (net, layer_list)
                # TUPLE that discriminator_F returns (lib/Teco.py:74) to tdiscrim_*_output, and the layer loss (:290) reads
                # real_layers / fake_layers that only the merged branch defines.  (Fix_margin, lib/Teco.py:283, is a constant
                # 0.0, not a flag: its hinge term is dead code in the reference.)
                raise ValueError("TecoGAN: only the merged spatio-temporal discriminator (Dt_mergeDs, config of record "
                                 "runGan.py:215) is built")
            t_size = 3 * (T // 3)
            t_gen_output = gen_outputs[:, :t_size].reshape(B * t_size, H, H, 3)
            t_targets = r_targets[:, :t_size].reshape(B * t_size, H, H, 3)
            t_batch = B * t_size // 3
            if not FLAGS.pingpang:  # :190-204 backward motion has to be calculated
                fb = torch.cat((r_inputs[:, 2:t_size:3], r_inputs[:, 1:t_size:3]), dim=-1).reshape(t_batch, crop, crop, 6)
                with variable_scope('fnet'):
                    flow_back_lr = fnet(fb, reuse=True)
                v_nxt = upscale_four(K.affine_act(flow_back_lr, 4.0, 0.0)).reshape(B, t_size // 3, H, H, 2)
                v_pre = gen_flow[:, 0:t_size:3]
            else:                   # :206-209 motion reused for the ping-pong sequence
                v_pre = gen_flow[:, 0:t_size:3]
                idx = list(range(T - 1))[-2:-1 - t_size:-3]
                v_nxt = torch.stack([gen_flow[:, i] for i in idx], dim=1)
            T_vel = torch.stack((v_pre, torch.zeros_like(v_pre), v_nxt), dim=2).reshape(B * t_size, H, H, 2).detach()
            if FLAGS.crop_dt < 1.0:  # :216-220
                crop_size_dt = int(crop * 4 * FLAGS.crop_dt)
                offset_dt = (crop * 4 - crop_size_dt) // 2
                crop_size_dt = crop * 4 - offset_dt * 2
                mask = torch.zeros((1, H, H, 1), device=r_inputs.device, dtype=torch.float32)
                mask[:, offset_dt:offset_dt + crop_size_dt, offset_dt:offset_dt + crop_size_dt] = 1.0

            def triplet9(x):   # [tb*3,h,w,3] -> [tb,h,w,9] = RRRGGGBBB over (t-1,t,t+1), :227-229
                hh, ww = x.shape[1], x.shape[2]
                return x.reshape(t_batch, 3, hh, ww, 3).permute(0, 2, 3, 4, 1).reshape(t_batch, hh, ww, 9)

            t_input = triplet9(r_inputs[:, :t_size].reshape(B * t_size, crop, crop, 3))
            input_hi = K.resize_bilinear(t_input.contiguous(), H, H)          # :240-244

            def dst_inputs(frames):   # :224-245 / :254-269
                warp = triplet9(K.dense_image_warp(frames.contiguous(), T_vel))
                if FLAGS.crop_dt < 1.0:
                    warp = warp * mask        # crop_to_bounding_box + tf.pad(CONSTANT): zero the unstable border
                return torch.cat((triplet9(frames), warp, input_hi), dim=-1)

            with variable_scope('tdiscriminator'):
                d_real, real_layers = discriminator_F(dst_inputs(t_targets), FLAGS=FLAGS)
                d_fake, fake_layers = discriminator_F(dst_inputs(t_gen_output), FLAGS=FLAGS)
            if FLAGS.D_LAYERLOSS:   # :275-313
                layer_norm = [12.0, 14.0, 24.0, 100.0]
                sum_layer_loss = 0
                lll = []
                for li in range(4):
                    ll = K.loss_l1(real_layers[li], fake_layers[li], per_pixel=True)
                    lll.append(ll)
                    sum_layer_loss = sum_layer_loss + 0.02 * ll / layer_norm[li]
                update_list += lll
                update_list_name += ["D_layer_%d_loss" % i for i in range(4)]
                update_list += [sum_layer_loss]
                update_list_name += ["D_layer_loss_sum"]

        # ---- generator losses (lib/Teco.py:316-390)
        content_loss = K.loss_l2(s_gen_output, s_targets)
        update_list += [content_loss]
        update_list_name += ["l2_content_loss"]
        gen_loss = content_loss
        warp_loss = K.loss_l2(input_frames.contiguous(), s_input_warp)
        update_list += [warp_loss]
        update_list_name += ["l2_warp_loss"]
        if vgg_on:
            vgg_loss = 0
            vl = []
            for name in VGG_LAYER_LABELS:
                d_ = K.loss_cosine(gen_vgg[name], target_vgg[name])
                vl.append(d_)
                vgg_loss = vgg_loss + d_
            gen_loss = gen_loss + FLAGS.vgg_scaling * vgg_loss
            update_list += vl + [vgg_loss]
            update_list_name += ["vgg_loss_%d" % (i + 2) for i in range(4)] + ["vgg_all"]
        if FLAGS.pingpang:
            first = gen_outputs[:, 0:RNN_N - 1].reshape(B * (RNN_N - 1), H, H, 3)
            last_rev = torch.flip(gen_outputs[:, RNN_N:], dims=(1,)).reshape(B * (RNN_N - 1), H, H, 3)
            pploss = K.loss_l1(first, last_rev, per_pixel=False)
            if FLAGS.pp_scaling > 0:
                gen_loss = gen_loss + pploss * FLAGS.pp_scaling
            update_list += [pploss]
            update_list_name += ["PingPang"]
        self.discrim_loss = None
        self.t_balance = None
        if GAN_Flag:
            gan = K.loss_gan(d_fake, d_real, FLAGS.EPS)
            t_adv = gan[0]
            gen_loss = gen_loss + FLAGS.ratio * t_adv * dt_ratio
            update_list += [t_adv]
            update_list_name += ["t_adversarial_loss"]
            if FLAGS.D_LAYERLOSS:
                gen_loss = gen_loss + sum_layer_loss * dt_ratio
            self.discrim_loss = gan[1]
            self.t_balance = gan[2] + t_adv                     # :399
            update_list += [gan[1], gan[3], gan[4]]
            update_list_name += ["t_discrim_loss", "t_discrim_real_output", "t_discrim_fake_output"]
        update_list += [gen_loss]
        update_list_name += ["All_loss_Gen"]
        self.gen_outputs, self.s_gen_output = gen_outputs, s_gen_output
        self.r_inputs, self.r_targets, self.gen_warppre = r_inputs, r_targets, gen_warppre   # the image summary's (:498-503)
        self.gen_loss = gen_loss
        self.fnet_loss = FLAGS.warp_scaling * warp_loss + gen_loss    # :443
        self.update_list, self.update_list_name = update_list, update_list_name
        self.dt_ratio = dt_ratio


class _FlatAdam:
    """tf.train.AdamOptimizer over one flat fp32 buffer (one fused kernel launch per step); the VariableStore
    entries become views of that buffer."""

    def __init__(self, store, names, lr, beta1, eps):
        self.names = list(names)
        n = sum(store[k].numel() for k in self.names)
        dev = store[self.names[0]].device if self.names else store.device
        self.flat = torch.empty(n, device=dev, dtype=torch.float32)
        self.m = torch.zeros_like(self.flat)
        self.v = torch.zeros_like(self.flat)
        self.views = {}
        o = 0
        for k in self.names:
            t = store[k]
            v = self.flat[o:o + t.numel()].view(t.shape)
            v.copy_(t)
            store[k] = v
            self.views[k] = (o, t.numel())
            o += t.numel()
        self.lr, self.b1, self.b2, self.eps, self.t = lr, beta1, 0.999, eps, 0
        self.n = n

    def step(self, flat_grad, lr, gscale=1.0):
        self.t += 1
        lr_t = lr * math.sqrt(1 - self.b2 ** self.t) / (1 - self.b1 ** self.t)
        K.adam_step(self.flat, self.m, self.v, flat_grad, lr_t, self.b1, self.b2, self.eps, gscale)


def _stack_scalars(vals, device):
    """Loss scalars (0-d tensors or Python numbers) as one fp32 device vector."""
    return torch.stack([v.detach().float() if torch.is_tensor(v) else torch.full((), float(v), device=device) for v in vals])


Network = collections.namedtuple('Network', 'gen_output, train, learning_rate, update_list, '
                                 'update_list_name, update_list_avg, image_summary, global_step')


class _TrainState:
    """Everything behind Network.train: three TF-Adams, loss EMA (decay .99, zero init), t_balance EMA and the
    adaptive-D branch (lib/Teco.py:415-496).  Under data parallelism (torch.distributed initialised) every rank runs
    its own clip shard and ONE all-reduce carries [G grads | FNet grads | D grads | t_balance | loss scalars]."""

    def __init__(self, r_inputs, r_targets, FLAGS, GAN_Flag):
        self.FLAGS, self.GAN = FLAGS, GAN_Flag
        self.static_in = r_inputs.detach().clone().contiguous()      # static buffers: the captured step reads these
        self.static_tg = r_targets.detach().clone().contiguous()
        self.use_graph = bool(getattr(FLAGS, 'train_cuda_graph', True))
        self.graph = None
        self.store = default_store()
        self.global_step = 0
        self.tb_ema = 0.0
        self.loss_ema = None
        self.counter1 = self.counter2 = 0
        self.last = None
        self.eval_in = self.eval_tg = self.eval_graph = None   # evaluate(): buffers and graph of its own
        self._summary_src = None
        self._gif = None
        from .. import config
        K.tc_cache_clear()                         # packed bf16 weights of a previous trainer are not ours
        prev_precision = config.precision()
        with torch.no_grad():                      # materialise every variable once (xavier / zeros / loaded values)
            config.set_precision("fp32")
            _Graph(r_inputs, r_targets, FLAGS, GAN_Flag, 0)
        config.set_precision(prev_precision)
        st = self.store
        g_names = [k for k in st if k.startswith('generator/')]
        f_names = [k for k in st if k.startswith('fnet/')]
        d_names = [k for k in st if k.startswith('tdiscriminator/')] if GAN_Flag else []
        lr, b1, eps = FLAGS.learning_rate, FLAGS.beta, FLAGS.adameps
        self.opt_g = _FlatAdam(st, g_names, lr, b1, eps)
        self.opt_f = _FlatAdam(st, f_names, lr, b1, eps)
        self.opt_d = _FlatAdam(st, d_names, lr, b1, eps) if d_names else None
        self.names = g_names + f_names + d_names
        self.n_scalars = 32
        self.bucket = torch.zeros(self.opt_g.n + self.opt_f.n + (self.opt_d.n if self.opt_d else 0) + self.n_scalars,
                                  device=st.device, dtype=torch.float32)
        st.touch()

    def learning_rate(self):
        F = self.FLAGS   # tf.train.exponential_decay (lib/Teco.py:97-98)
        p = self.global_step / float(F.decay_step)
        if F.stair:
            p = math.floor(p)
        return F.learning_rate * (F.decay_rate ** p)

    def _compute(self):
        """Forward over the unrolled recurrence, every loss, backward, and the flat bucket
        [G grads | FNet grads | D grads | t_balance | loss scalars] -- no host synchronisation, so the whole thing can be
        captured in one CUDA graph (about 2000 kernel launches for case 4, 6000 for case 3)."""
        from .. import config
        K.tc_cache_clear()
        F = self.FLAGS
        st = self.store
        leaves = {k: st[k].detach().requires_grad_(True) for k in self.names}   # fresh leaf views of the flat buffers
        saved = {k: st[k] for k in self.names}
        for k in self.names:
            st[k] = leaves[k]
        prev_precision = config.precision()
        try:
            config.set_precision("fp32")
            g = _Graph(self.static_in, self.static_tg, F, self.GAN, self.global_step)
            gf = self.opt_g.names + self.opt_f.names
            grads = torch.autograd.grad(g.fnet_loss, [leaves[k] for k in gf], retain_graph=self.GAN, allow_unused=True)
            d_grads = ()
            if self.GAN:
                d_grads = torch.autograd.grad(g.discrim_loss, [leaves[k] for k in self.opt_d.names], allow_unused=True)
        finally:
            config.set_precision(prev_precision)
            for k in self.names:
                st[k] = saved[k]
        b = self.bucket
        o = 0
        for k, gr in zip(gf + (self.opt_d.names if self.GAN else []), list(grads) + list(d_grads)):
            n = st[k].numel()
            if gr is None:
                b[o:o + n].zero_()
            else:
                b[o:o + n].copy_(gr.reshape(-1))
            o += n
        scal = _stack_scalars([g.t_balance if self.GAN else torch.zeros((), device=b.device)] + list(g.update_list), b.device)
        b[o:o + scal.numel()].copy_(scal)
        self._scal_off, self._n_scal = o, scal.numel()
        self._names_now = g.update_list_name
        self._gen_outputs = g.gen_outputs.detach()
        self._summary_src = (g.r_inputs, g.r_targets, self._gen_outputs, [w.detach() for w in g.gen_warppre])

    def __call__(self, r_inputs=None, r_targets=None):
        F = self.FLAGS
        if r_inputs is not None:
            self.static_in.copy_(r_inputs)
            self.static_tg.copy_(r_targets)
        if self.use_graph and F.Dt_ratio_add == 0.0:
            if self.graph is None:
                # warm-up on a side stream (lazy initialisations, allocator), then capture the whole step once
                side = torch.cuda.Stream()
                side.wait_stream(torch.cuda.current_stream())
                with torch.cuda.stream(side):
                    self._compute()
                torch.cuda.current_stream().wait_stream(side)
                torch.cuda.synchronize()
                self.graph = torch.cuda.CUDAGraph()
                with torch.cuda.graph(self.graph):
                    self._compute()
            self.graph.replay()
        else:
            self._compute()
        b, o = self.bucket, self._scal_off
        from ..parallel import allreduce_bucket, decide_with_d
        inv = allreduce_bucket(b)                   # the single NCCL all-reduce of the step (sum); inv = 1/world
        scal_host = (b[o:o + self._n_scal] * inv).tolist()       # one small D2H: drives the tb < Dbalance branch + logging
        lr = self.learning_rate()
        ng, nf = self.opt_g.n, self.opt_f.n
        with_d = False
        if self.GAN:
            with_d, self.tb_ema = decide_with_d(self.tb_ema, scal_host[0], F.Dbalance)   # lib/Teco.py:464,477,494
            if with_d:
                self.opt_d.step(b[ng + nf:ng + nf + self.opt_d.n], lr, inv)
                self.counter1 += 1
            else:
                self.counter2 += 1
        self.opt_g.step(b[0:ng], lr, inv)
        self.opt_f.step(b[ng:ng + nf], lr, inv)
        self.store.touch()
        vals = scal_host[1:]
        if self.loss_ema is None:
            self.loss_ema = [0.0] * len(vals)
        self.loss_ema = [0.99 * a_ + 0.01 * v for a_, v in zip(self.loss_ema, vals)]
        self.global_step += 1
        self.last = {"update_list": vals, "update_list_name": self._names_now, "with_d": with_d, "lr": lr,
                     "gen_outputs": self._gen_outputs, "t_balance": scal_host[0], "tb_ema": self.tb_ema}
        return self.last

    # ---- forward-only evaluation (reference main.py:299-304,391-402: the validation fetch of Net.update_list) -------
    def _evaluate_compute(self):
        """The training graph's forward on eval_in / eval_tg with the current weights: the kernels, precision and packed-weight
        discipline of _compute, no autograd tape, and nothing written but the tensors this pass allocates."""
        from .. import config
        K.tc_cache_clear()            # pack the current weights in this pass (inside this graph when captured)
        prev_precision = config.precision()
        try:
            config.set_precision("fp32")
            with torch.no_grad(), config.train_forward():
                g = _Graph(self.eval_in, self.eval_tg, self.FLAGS, self.GAN, self.global_step)
        finally:
            config.set_precision(prev_precision)
        self._eval_scal = _stack_scalars(g.update_list, self.eval_in.device)
        self._eval_names = list(g.update_list_name)

    def evaluate(self, r_inputs, r_targets):
        """Losses of the training graph on another batch, without training: {name: float} for every entry of
        Network.update_list (the reference's `uplen` names -- t_balance, Dst_ratio and the D counters are running state,
        not losses of a batch).  Runs at the current global_step (the Dst ratio of the last step) on the kernels of
        training, from input buffers and a CUDA graph of its own, captured under the rule of the training step.  Weights,
        Adam moments, the step counters, the EMAs, the with-D decision and the training step's buffers are only read."""
        if self.eval_in is None:
            self.eval_in = torch.empty_like(self.static_in)
            self.eval_tg = torch.empty_like(self.static_tg)
        self.eval_in.copy_(r_inputs)
        self.eval_tg.copy_(r_targets)
        if self.use_graph and self.FLAGS.Dt_ratio_add == 0.0:
            if self.eval_graph is None:
                side = torch.cuda.Stream()
                side.wait_stream(torch.cuda.current_stream())
                with torch.cuda.stream(side):
                    self._evaluate_compute()
                torch.cuda.current_stream().wait_stream(side)
                torch.cuda.synchronize()
                self.eval_graph = torch.cuda.CUDAGraph()
                with torch.cuda.graph(self.eval_graph):
                    self._evaluate_compute()
            self.eval_graph.replay()
        else:
            self._evaluate_compute()
        return dict(zip(self._eval_names, self._eval_scal.tolist()))

    # ---- GIF image summaries (reference lib/Teco.py:498-503, lib/ops.py:434-484) -------------------------------------
    def image_summary(self):
        """The reference's four GIF summaries of the last training step's own batch and forward pass (the weights before
        that step's update): [(tag, height, width, GIF bytes)] for LR = r_inputs, HR = deprocess(r_targets), Generated =
        deprocess(gen_outputs) and WarpPreGen = deprocess(the T - 1 warped previous outputs), each the first
        min(4, batch_size) clips of the step (ping-pong extended with --pingpang), quantised as
        tf.image.convert_image_dtype(saturate=True).  Tags image_summaries/<name>/gif/<i>, or .../gif when one clip is
        written.  Quantisation and the four encodes run on the device; the host waits for them together."""
        if self._summary_src is None:
            raise RuntimeError("image_summary: no training step has run yet")
        from ..gif import GifEncoder, convert_image_u8
        from .._encode import collect
        lr, hr, gen, warppre = self._summary_src
        k = min(4, self.FLAGS.batch_size)
        if self._gif is None:
            self._gif = {name: GifEncoder("image_summary " + name) for name in ("LR", "HR", "Generated", "WarpPreGen")}
        srcs = (("LR", lr[:k], False), ("HR", hr[:k], True), ("Generated", gen[:k], True),
                ("WarpPreGen", torch.stack([w[:k] for w in warppre], dim=1), True))
        pending, shapes = [], []
        for name, x, dep in srcs:
            u8 = convert_image_u8(x, deprocess=dep)
            pending.append(self._gif[name].launch(u8))
            shapes.append((name, int(u8.shape[2]), int(u8.shape[3])))
        out = []
        for (name, h, w), files in zip(shapes, collect(pending)):
            for i, data in enumerate(files):
                tag = "image_summaries/%s/gif" % name + ("" if k == 1 else "/%d" % i)
                out.append((tag, h, w, data))
        return out

    # ---- checkpoint / resume (reference: tf.train.Saver over GLOBAL_VARIABLES, main.py:307,346-349) -------------------
    def state_tensors(self):
        """Everything besides the model variables that a resumed run needs, as {name: CPU tensor}.  Adam moments use
        TensorFlow's slot names (`<variable>/Adam` = m, `<variable>/Adam_1` = v), `global_step` is the Saver's; the rest
        (per-optimiser step counts, which TF keeps as beta powers, and the EMAs of lib/Teco.py:415-423,455-461) lives
        under `teco_b200/`."""
        out = {"global_step": torch.tensor(self.global_step, dtype=torch.int64)}
        for tag, opt in (("g", self.opt_g), ("f", self.opt_f), ("d", self.opt_d)):
            if opt is None:
                continue
            for k, (o, n) in opt.views.items():
                shape = self.store[k].shape
                out[k + "/Adam"] = opt.m[o:o + n].view(shape).detach().cpu().clone()
                out[k + "/Adam_1"] = opt.v[o:o + n].view(shape).detach().cpu().clone()
            out["teco_b200/adam_steps_" + tag] = torch.tensor(opt.t, dtype=torch.int64)
        out["teco_b200/tb_ema"] = torch.tensor(self.tb_ema, dtype=torch.float64)
        out["teco_b200/loss_ema"] = torch.tensor(self.loss_ema or [], dtype=torch.float64)
        out["teco_b200/d_counters"] = torch.tensor([self.counter1, self.counter2], dtype=torch.int64)
        return out

    def load_state(self, get):
        """Inverse of state_tensors.  `get(name)` returns an array-like or None; Adam slots are also looked up by the
        suffix TensorFlow may have produced (`<optimizer scope>/<variable>/Adam`).  Missing pieces keep their fresh
        values (moments 0, counters 0) and are reported in the returned list."""
        missing = []

        def fetch(name):
            v = get(name)
            if v is None:
                missing.append(name)
                return None
            return torch.as_tensor(v)
        gs = fetch("global_step")
        if gs is not None:
            self.global_step = int(gs)
        for tag, opt in (("g", self.opt_g), ("f", self.opt_f), ("d", self.opt_d)):
            if opt is None:
                continue
            for k, (o, n) in opt.views.items():
                for slot, buf in (("/Adam", opt.m), ("/Adam_1", opt.v)):
                    v = fetch(k + slot)
                    if v is not None:
                        if v.numel() != n:
                            raise ValueError('Wrong shape in for {} in ckpt,expected {}, got {}.'.format(
                                k + slot, str(tuple(self.store[k].shape)), str(tuple(v.shape))))
                        buf[o:o + n].copy_(v.reshape(-1).to(dtype=torch.float32))
            t = fetch("teco_b200/adam_steps_" + tag)
            opt.t = int(t) if t is not None else self._tf_adam_steps(get, tag, opt)
        v = fetch("teco_b200/tb_ema")
        if v is not None:
            self.tb_ema = float(v)
        v = fetch("teco_b200/loss_ema")
        if v is not None and v.numel():
            self.loss_ema = [float(x) for x in v.reshape(-1)]
        v = fetch("teco_b200/d_counters")
        if v is not None:
            self.counter1, self.counter2 = int(v[0]), int(v[1])
        else:                                   # a reference checkpoint keeps them as graph variables (lib/Teco.py:456-459)
            c1, c2 = get("generator_train/gen_train_with_D_counter"), get("generator_train/gen_train_wo_D_counter")
            if c1 is not None and c2 is not None:
                self.counter1, self.counter2 = int(torch.as_tensor(c1)), int(torch.as_tensor(c2))
        return missing

    def _tf_adam_steps(self, get, tag, opt):
        """Step count of one optimiser when resuming from a checkpoint written by the REFERENCE.  TensorFlow keeps it as
        beta1_power = beta1^(t+1) (AdamOptimizer._finish multiplies after every apply).  All three apply_gradients calls sit
        in variable_scope('generator_train') (lib/Teco.py:438-481), created in the order discriminator, generator, fnet inside
        train_gen_withD, hence the suffixes.  The generator and fnet step every iteration (= global_step); the discriminator
        only when t_balance < Dbalance, i.e. gen_train_with_D_counter times (lib/Teco.py:456,464)."""
        import math
        suffix = {"d": "", "g": "_1", "f": "_2"} if self.GAN else {"g": "", "f": "_1"}
        bp = get("generator_train/beta1_power" + suffix.get(tag, ""))
        if bp is not None and 0.0 < float(torch.as_tensor(bp)) < 1.0 and 0.0 < opt.b1 < 1.0:
            return max(0, int(round(math.log(float(torch.as_tensor(bp))) / math.log(opt.b1))) - 1)
        if tag == "d":
            c1 = get("generator_train/gen_train_with_D_counter")
            if c1 is not None:
                return int(torch.as_tensor(c1))
        return self.global_step

    def update_list_avg(self):
        avg = list(self.loss_ema or [])
        if self.GAN:
            avg += [self.tb_ema, min(self.FLAGS.Dt_ratio_max, self.FLAGS.Dt_ratio_0 + self.FLAGS.Dt_ratio_add * self.global_step),
                    self.counter1, self.counter2]
        return avg


def TecoGAN(r_inputs, r_targets, FLAGS, GAN_Flag=True):
    """reference lib/Teco.py:77-517.  r_inputs [b,frame,h,w,3] in [0,1], r_targets [b,frame,4h,4w,3] in [-1,1]."""
    state = _TrainState(r_inputs, r_targets, FLAGS, GAN_Flag)
    from .. import config
    prev_precision = config.precision()
    config.set_precision("fp32")
    with torch.no_grad():
        g0 = _Graph(r_inputs, r_targets, FLAGS, GAN_Flag, 0)
    config.set_precision(prev_precision)
    names = list(g0.update_list_name)
    if GAN_Flag:
        names_avg = names + ["t_balance", "Dst_ratio", "withD_counter", "w_o_D_counter"]
    else:
        names_avg = names
    return Network(
        gen_output=g0.s_gen_output,
        train=state,
        learning_rate=state.learning_rate,
        update_list=[float(v) for v in g0.update_list],
        update_list_name=names_avg,
        update_list_avg=state.update_list_avg,
        image_summary=state.image_summary,
        global_step=lambda: state.global_step,
    )


def FRVSR(r_inputs, r_targets, FLAGS):
    """reference lib/Teco.py:521-522"""
    return TecoGAN(r_inputs, r_targets, FLAGS, False)
