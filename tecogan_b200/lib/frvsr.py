"""Mirror of the reference's lib/frvsr.py: fnet (flow estimator) and generator_F (SRNet).

Two execution modes, chosen by tecogan_b200.config:
  * "fp32": every layer through the fp32 CUDA-core kernels, differentiable (training, exact parity);
  * "bf16": NHWC bf16 activations through the wgmma tensor-core kernel (inference hot path).
"""
import torch

from .. import config
from .ops import (ACT_LRELU02, ACT_RELU, ACT_TANH24, bicubic_four, conv2, conv2_tran, maxpool, preprocess)
from .. import kernels as K
from ..variables import variable_scope


def fnet(fnet_input, reuse=False):
    """reference lib/frvsr.py:4-41.  [n,h,w,6] (prev RGB ++ cur RGB in [0,1]) -> flow [n,8*(h//8),8*(w//8),2]."""
    if config.use_tensor_cores() and not torch.is_grad_enabled():
        from ..tc_nets import fnet_tc
        with variable_scope('autoencode_unit', reuse=reuse):
            return fnet_tc(fnet_input)

    def down_block(inputs, output_channel=64, stride=1, scope='down_block'):
        with variable_scope(scope):
            net = conv2(inputs, 3, output_channel, stride, use_bias=True, scope='conv_1', act=ACT_LRELU02)
            net = conv2(net, 3, output_channel, stride, use_bias=True, scope='conv_2', act=ACT_LRELU02)
            net = maxpool(net)
        return net

    def up_block(inputs, output_channel=64, stride=1, scope='up_block'):
        with variable_scope(scope):
            net = conv2(inputs, 3, output_channel, stride, use_bias=True, scope='conv_1', act=ACT_LRELU02)
            net = conv2(net, 3, output_channel, stride, use_bias=True, scope='conv_2', act=ACT_LRELU02)
            net = K.resize_bilinear(net, net.shape[1] * 2, net.shape[2] * 2)
        return net

    with variable_scope('autoencode_unit', reuse=reuse):
        net = down_block(fnet_input, 32, scope='encoder_1')
        net = down_block(net, 64, scope='encoder_2')
        net = down_block(net, 128, scope='encoder_3')
        net = up_block(net, 256, scope='decoder_1')
        net = up_block(net, 128, scope='decoder_2')
        net1 = up_block(net, 64, scope='decoder_3')
        with variable_scope('output_stage'):
            net = conv2(net1, 3, 32, 1, scope='conv1', act=ACT_LRELU02)
            net = conv2(net, 3, 2, 1, scope='conv2', act=ACT_TANH24)  # tanh(x)*24: max velocity, lib/frvsr.py:39
    return net


def generator_F(gen_inputs, gen_output_channels, reuse=False, FLAGS=None):
    """reference lib/frvsr.py:44-88.  gen_inputs [B,h,w,51] = LR RGB (3) ++ space-to-depth of the warped previous
    HR frame (48), all in [0,1]  ->  HR [B,4h,4w,3] in ~[-1,1]."""
    if FLAGS is None:
        raise ValueError('No FLAGS is provided for generator')
    if config.use_tensor_cores() and not torch.is_grad_enabled():
        from ..tc_nets import generator_tc
        with variable_scope('generator_unit', reuse=reuse):
            return generator_tc(gen_inputs, gen_output_channels, FLAGS.num_resblock)

    def residual_block(inputs, output_channel=64, stride=1, scope='res_block'):
        with variable_scope(scope):
            net = conv2(inputs, 3, output_channel, stride, use_bias=True, scope='conv_1', act=ACT_RELU)
            net = conv2(net, 3, output_channel, stride, use_bias=True, scope='conv_2', res=inputs)
        return net

    with variable_scope('generator_unit', reuse=reuse):
        with variable_scope('input_stage'):
            net = conv2(gen_inputs, 3, 64, 1, scope='conv', act=ACT_RELU)
        for i in range(1, FLAGS.num_resblock + 1, 1):
            net = residual_block(net, 64, 1, 'resblock_%d' % (i))
        with variable_scope('conv_tran2highres'):
            net = conv2_tran(net, 3, 64, 2, scope='conv_tran1', act=ACT_RELU)
            net = conv2_tran(net, 3, 64, 2, scope='conv_tran2', act=ACT_RELU)
        with variable_scope('output_stage'):
            low_res_in = gen_inputs[:, :, :, 0:3]
            bicubic_hi = bicubic_four(low_res_in.contiguous())
            net = conv2(net, 3, gen_output_channels, 1, scope='conv', res=bicubic_hi)
            net = preprocess(net)
    return net
