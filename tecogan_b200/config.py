"""Run-time configuration of the compute path (not part of the reference interface)."""
import contextlib as _contextlib
import os as _os

_cfg = {"precision": "bf16", "train_precision": "fp32", "lin_trunk": {"1": True, "0": False}.get(_os.environ.get("TECO_LIN_TRUNK")),
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
    """32x32 frames (the metric configuration's LR clips): whether the generator's input conv + residual blocks run as ONE
    launch that keeps each clip's activations in shared memory (teco_conv3x3_lin_tc; a cluster of two CTAs owns a clip
    through all 33 layers) instead of 33 per-layer launches.  None (the default, or TECO_LIN_TRUNK unset): automatic, the
    one launch when the batch fills at least LIN_TRUNK_MIN_FILL of the rounds of G clusters it needs (G: clusters resident
    at once, 66 on an H100 SXM), where it measured faster; True / False (TECO_LIN_TRUNK=1 / 0) force it on (for batches of
    at least 8 clips) or off."""
    _cfg["lin_trunk"] = None if on is None else bool(on)


def lin_trunk():
    return _cfg["lin_trunk"]


# A round of the one-launch trunk takes about as long whether it holds 1 or G clips, while the per-layer launches scale
# with the batch: on an H100 SXM (700 W) the one launch was 1.20-1.32x faster at 66, 132, 198 and 264 clips (full rounds)
# and 0.71-0.81x at 8 and 67 (1 / 8 and 1 / 2 of a round used); see tools/ab_trunk.py and DESIGN 4.1b.
LIN_TRUNK_MIN_FILL = 0.8


def train_tc_all():
    """bf16 training mode: also run conv2_tran (forward, input and weight gradient), the narrow-output convolutions
    (generator 64 -> 3, fnet 32 -> 2) and the discriminator's 4x4 stride-2 convolutions on wgmma instead of the fp32
    kernels (TECO_TRAIN_TC_ALL=0 restores the latter)."""
    return _cfg["train_tc_all"]
