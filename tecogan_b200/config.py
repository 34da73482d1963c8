"""Run-time configuration of the compute path (not part of the reference interface)."""
import contextlib as _contextlib

_cfg = {"precision": "bf16", "train_precision": "fp32", "train_forward": False, "deterministic": False}


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
    """'fp32' (default, exact parity with the oracle) or 'bf16': the training graph's 3x3 stride-1 convolutions (the
    narrow-output generator 64 -> 3 and fnet 32 -> 2 included), conv2_tran and the discriminator's 4x4 stride-2
    convolutions run forward, input and weight gradient on wgmma kernels wherever their shapes and activations fit (bf16
    operands, fp32 accumulation, fp32 master weights; lib/ops.py conv2 / conv2_tran)."""
    if p not in ("bf16", "fp32"):
        raise ValueError("train precision must be 'bf16' or 'fp32'")
    _cfg["train_precision"] = p


def train_precision():
    return _cfg["train_precision"]


def set_deterministic(on):
    """True: every reduction of the training path (weight, bias and batch-norm gradients, batch-norm statistics, loss
    scalars, the warp and resize scatter gradients, the multi-GPU gradient sum) runs on the fixed-order *_det kernels,
    whose summation order depends on the shapes alone, so one seed gives bit-identical runs on one GPU model and build.
    False (default): the atomic kernels."""
    _cfg["deterministic"] = bool(on)


def deterministic():
    return _cfg["deterministic"]


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
