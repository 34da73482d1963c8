"""Mirror of the reference's lib/ops.py op wrappers (the ones on the hot path, SURVEY.md section 2 row 8).
Every function keeps the reference name and argument meaning; arithmetic runs in libteco.so kernels."""
import numpy as np
import torch

from .. import config
from .. import kernels as K
from .._ffi import ACT_NONE, ACT_RELU, ACT_LRELU02, ACT_TANH24, ACT_SIGMOID  # noqa: F401
from ..variables import get_variable, variable_scope


def preprocess(image):
    """[0,1] -> [-1,1]   (reference lib/ops.py:13-16)"""
    return K.affine_act(image, 2.0, -1.0)


def deprocess(image):
    """[-1,1] -> [0,1]   (reference lib/ops.py:19-22)"""
    return K.affine_act(image, 0.5, 0.5)


def preprocessLR(image):
    """identity (reference lib/ops.py:25-27)"""
    return image


def deprocessLR(image):
    """identity (reference lib/ops.py:30-32)"""
    return image


def conv2_tran(batch_input, kernel=3, output_channel=64, stride=1, use_bias=True, scope='conv', act=ACT_NONE):
    """slim.conv2d_transpose(.., [k,k], stride, 'SAME', NHWC, activation_fn=None), xavier init, zero bias
    (reference lib/ops.py:35-44).  Variables: <scope>/Conv2d_transpose/{weights[k,k,Cout,Cin], biases}.
    `act` is an extension: fuse the activation the caller applies next."""
    if kernel != 3 or stride != 2:
        raise ValueError("conv2_tran: only the 3x3 stride-2 configuration of the reference (lib/frvsr.py:73,76) is built")
    cin = batch_input.shape[-1]
    with variable_scope(scope), variable_scope('Conv2d_transpose'):
        w = get_variable('weights', (kernel, kernel, output_channel, cin),
                         fans=(kernel * kernel * output_channel, kernel * kernel * cin))
        b = get_variable('biases', (output_channel,), init='zeros') if use_bias else None
    if (torch.is_grad_enabled() and config.train_precision() == "bf16" and config.train_tc_all() and cin == 64 and output_channel == 64
            and act in (ACT_NONE, ACT_RELU, ACT_LRELU02)):
        return K.conv_transpose2x_train_tc(batch_input, w, b, act)   # wgmma forward, input and weight gradients
    return K.conv2d_transpose(batch_input, w, b, act)


def conv2(batch_input, kernel=3, output_channel=64, stride=1, use_bias=True, scope='conv', act=ACT_NONE, res=None):
    """slim.conv2d(.., [k,k], stride, 'SAME', NHWC, activation_fn=None), xavier init, zero bias
    (reference lib/ops.py:47-56).  Variables: <scope>/Conv/{weights[k,k,Cin,Cout], biases}.
    Extensions: `act` fuses the following activation, `res` adds a residual after the convolution."""
    cin = batch_input.shape[-1]
    with variable_scope(scope), variable_scope('Conv'):
        w = get_variable('weights', (kernel, kernel, cin, output_channel),
                         fans=(kernel * kernel * cin, kernel * kernel * output_channel))
        b = get_variable('biases', (output_channel,), init='zeros') if use_bias else None
    if (kernel == 3 and stride == 1 and torch.is_grad_enabled() and config.train_precision() == "bf16"
            and (output_channel >= 16 or config.train_tc_all())
            and (act in (ACT_NONE, ACT_RELU, ACT_LRELU02) or (act == ACT_TANH24 and output_channel < 16 and res is None))):
        return K.conv3x3_train_tc(batch_input, w, b, act, res)      # wgmma forward, input and weight gradients
    return K.conv2d(batch_input, w, b, stride, act, res)


def lrelu(inputs, alpha):
    """keras LeakyReLU (reference lib/ops.py:84-85); the path only ever uses alpha = 0.2."""
    if abs(alpha - 0.2) > 1e-12:
        raise ValueError("lrelu: only alpha=0.2 (the reference's value) is built")
    return K.affine_act(inputs, 1.0, 0.0, ACT_LRELU02)


def relu(inputs):
    """tf.nn.relu (reference lib/frvsr.py:53,63,74,77)"""
    return K.affine_act(inputs, 1.0, 0.0, ACT_RELU)


def batchnorm(inputs, is_training, lrelu02=False):
    """slim.batch_norm(decay=.9, eps=1e-3, scale=False, fused=True, is_training) -- reference lib/ops.py:88-90.
    Variables: BatchNorm/beta (moving stats are never read by any forward of the reference: SURVEY A.10)."""
    if not is_training:
        raise ValueError("batchnorm: the reference always calls it with is_training=True (lib/Teco.py:38)")
    c = inputs.shape[-1]
    with variable_scope('BatchNorm'):
        beta = get_variable('beta', (c,), init='zeros')
    return K.batchnorm_train(inputs, beta, lrelu02)


def maxpool(inputs, scope='maxpool'):
    """slim.max_pool2d(inputs, [2,2]) (reference lib/ops.py:92-93)"""
    return K.maxpool2(inputs)


def denselayer(inputs, output_size):
    """tf.layers.Dense on the channel axis, with bias (reference lib/ops.py:96-103) == 1x1 convolution.
    Variables: dense/{kernel[Cin,out], bias[out]}."""
    cin = inputs.shape[-1]
    with variable_scope('dense'):
        kern = get_variable('kernel', (cin, output_size), fans=(cin, output_size))
        bias = get_variable('bias', (output_size,), init='zeros')
    return K.conv2d(inputs, kern.view(1, 1, cin, output_size), bias, 1, ACT_NONE, None)


def upscale_four(inputs, scope='upscale_four'):
    """legacy bilinear x4 (reference lib/ops.py:126-163)"""
    return K.resize_bilinear(inputs, inputs.shape[1] * 4, inputs.shape[2] * 4)


def bicubic_four(inputs, scope='bicubic_four'):
    """x4 Keys bicubic A=-0.75 (reference lib/ops.py:166-212).  No gradient: its only use is on the LR input."""
    return K.bicubic4(inputs.detach())


def tf_data_gaussDownby4(HRdata, sigma=1.5):
    """9x9 sigma-1.5 Gaussian, stride 4, VALID (reference lib/ops.py:347-367)"""
    if abs(sigma - 1.5) > 1e-12:
        raise ValueError("tf_data_gaussDownby4: only sigma=1.5 (the reference's value) is built")
    return K.gauss_down4(HRdata)


def save_img(out_path, img):
    """clip(img*255) -> uint8 -> BGR imwrite (reference lib/ops.py:521-523).  img: [H,W,3] CUDA or numpy in [0,1]."""
    import cv2 as cv
    if torch.is_tensor(img):
        img = K.to_u8(img).cpu().numpy()
    else:
        img = np.clip(img * 255.0, 0, 255).astype(np.uint8)
    cv.imwrite(out_path, img[:, :, ::-1])
