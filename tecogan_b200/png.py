"""PNG encoding on the GPU: the bytes cv2.imwrite writes for the same frame (libpng, filter Sub, zlib level 1 with the
run-length strategy), computed by tecogan_b200/csrc/png.cu.  DESIGN.md section 4.5.

encode_png(frame) takes a contiguous [H, W, 3] uint8 CUDA tensor in RGB order and returns the file's bytes.  The
workspace, the device output and the pinned host buffer are kept for the last frame size and device, so a sequence of
equal-sized frames allocates nothing after its first frame.
"""
from ._encode import FrameEncoder

_encoder = FrameEncoder("teco_png", "encode_png")
_state = _encoder.state


def plan_bytes(h, w):
    """(workspace bytes, output capacity) for an h x w frame; ValueError for sizes the encoder does not take."""
    return _encoder.plan_bytes(h, w)


def encode_png(frame_u8):
    """[H, W, 3] uint8 RGB CUDA tensor -> bytes of the PNG file cv2.imwrite writes for its BGR copy."""
    return _encoder.encode(frame_u8)
