"""Run-time configuration of the compute path (not part of the reference interface)."""
import contextlib as _contextlib
import os as _os

_cfg = {"precision": "bf16", "train_precision": "fp32", "lin_trunk": _os.environ.get("TECO_LIN_TRUNK", "0") == "1",
        "train_tc_all": _os.environ.get("TECO_TRAIN_TC_ALL", "1") == "1", "train_forward": False}


def set_precision(p):
    """'bf16': wgmma tensor-core convolutions for inference (default); 'fp32': CUDA-core fp32 everywhere."""
    if p not in ("bf16", "fp32"):
        raise ValueError("precision must be 'bf16' or 'fp32'")
    _cfg["precision"] = p


def precision():
    return _cfg["precision"]


def use_tensor_cores():
    return _cfg["precision"] == "bf16"


def set_train_precision(p):
    """'fp32' (default, exact parity with the oracle) or 'bf16': 3x3 stride-1 convolutions of the training graph run
    forward + input-gradient on the wgmma kernel (bf16 operands, fp32 accumulation, fp32 master weights)."""
    if p not in ("bf16", "fp32"):
        raise ValueError("train precision must be 'bf16' or 'fp32'")
    _cfg["train_precision"] = p


def train_precision():
    return _cfg["train_precision"]


@_contextlib.contextmanager
def train_forward():
    """Inside this block the training graph picks its convolution kernels as under autograd even when gradients are off:
    the trainer's forward-only evaluation (Network.train.evaluate) runs under torch.no_grad() on the kernels a training
    step runs, so its losses are the ones training would report for the same batch."""
    prev = _cfg["train_forward"]
    _cfg["train_forward"] = True
    try:
        yield
    finally:
        _cfg["train_forward"] = prev


def training_kernels(grad_enabled):
    """Convolution dispatch of the training graph: its kernels run under autograd and inside train_forward()."""
    return grad_enabled or _cfg["train_forward"]


def set_lin_trunk(on):
    """32-pixel-wide frames (the metric configuration's 32x32 LR clips): run the generator's input conv + all residual
    blocks as ONE launch of the multi-layer chain kernel (teco_conv3x3_lin_tc; every CTA keeps its own clips for all
    layers), for batches of at least 8 clips.  Off by default: on an H100 the 33 per-layer launches are faster at every
    batch measured (8 to 264 clips: 1.4x to 7.6x) -- both have one CTA per SM in flight, but the chain's CTA owns whole
    images through all 33 layers while the per-layer kernel spreads each layer's small tiles over every SM -- so bench.py
    times the chain next to them instead."""
    _cfg["lin_trunk"] = bool(on)


def lin_trunk():
    return _cfg["lin_trunk"]


def train_tc_all():
    """bf16 training mode: also run conv2_tran (forward, input and weight gradient) and the narrow-output convolutions
    (generator 64 -> 3, fnet 32 -> 2) on wgmma instead of the fp32 kernels (TECO_TRAIN_TC_ALL=0 restores the latter)."""
    return _cfg["train_tc_all"]
