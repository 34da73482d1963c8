"""GIF encoding on the GPU for the TensorBoard image summaries of training (reference lib/Teco.py:498-503,
lib/ops.py:399-431), computed by tecogan_b200/csrc/gif.cu.  DESIGN.md section 4.8.

encode_gif(frames) takes a contiguous [N, T, H, W, 3] uint8 CUDA tensor in RGB order (T >= 1, 1 <= H, W <= 65535) and
returns N GIF89a files: one looping animation at 3 fps per clip, its palette a median cut of up to 256 colours over all of
its frames, Sierra-2-4A error diffusion per frame.  An animation of at most 256 distinct colours decodes to its input
exactly.  The bytes are not ffmpeg's (the reference's encoder); every rule is specified in DESIGN.md so they can be
pinned.  A GifEncoder keeps its buffers for the last batch size and device; encode_gif uses one module-wide encoder.

convert_image_u8(x, deprocess) is the reference's summary quantisation, tf.image.convert_image_dtype(x, tf.uint8,
saturate=True) of a float32 tensor, after deprocess ((x + 1) / 2) when asked.
"""
import torch

from ._encode import FrameEncoder, check_rgb8, collect
from ._ffi import call, lib, ptr, stream_ptr

MAX_SIDE = 65535
FPS = 3


class GifEncoder(FrameEncoder):
    def __init__(self, name="encode_gif"):
        super().__init__("teco_gif", name)

    def launch(self, frames_u8):
        """Enqueue the encode of a [N, T, H, W, 3] batch on the current stream; collect() the result."""
        check_rgb8(frames_u8, self.name, "batch", "N, T, H, W")
        n, t, h, w = (int(d) for d in frames_u8.shape[:4])
        if t < 1 or n < 1 or not (1 <= h <= MAX_SIDE and 1 <= w <= MAX_SIDE):
            raise ValueError("%s: bad animation batch %s (N, T >= 1, 1 <= H, W <= %d)"
                             % (self.name, tuple(frames_u8.shape), MAX_SIDE))
        return super().launch(frames_u8, (n, t, h, w), n)

    def encode(self, frames_u8):
        """[N, T, H, W, 3] uint8 RGB CUDA tensor -> list of N GIF files (bytes)."""
        return collect([self.launch(frames_u8)])[0]


_encoder = GifEncoder()
_state = _encoder.state


def plan_bytes(n, t, h, w):
    """(workspace bytes, output capacity) for N animations of T frames of h x w; ValueError for sizes not taken."""
    return _encoder.plan_bytes(n, t, h, w)


def encode_gif(frames_u8):
    """[N, T, H, W, 3] uint8 RGB CUDA tensor -> list of N GIF89a files (bytes), one animation per clip."""
    return _encoder.encode(frames_u8)


def convert_image_u8(x, deprocess=False):
    """float32 CUDA tensor -> uint8 tensor of its shape: trunc(clamp(x' * 255.5, 0, 255)) with x' = (x + 1) / 2 when
    `deprocess`, else x (NaN -> 0), in float32 as tf.image.convert_image_dtype(saturate=True) computes it."""
    if not torch.is_tensor(x) or x.dtype != torch.float32 or not x.is_cuda:
        raise ValueError("convert_image_u8: expected a float32 CUDA tensor")
    x = x.contiguous()
    y = torch.empty(x.shape, dtype=torch.uint8, device=x.device)
    if x.numel():
        lib()
        with torch.cuda.device(x.device):
            call("teco_convert_image_u8", ptr(x), ptr(y), x.numel(), int(bool(deprocess)), stream_ptr())
    return y
