"""JPEG encoding on the GPU: the bytes cv2.imwrite writes for the same frame with cv2's defaults (baseline, quality 95,
4:2:0, islow FDCT, the Annex K Huffman tables), computed by tecogan_b200/csrc/jpeg.cu.  DESIGN.md section 4.6.

encode_jpeg(frame) takes a contiguous [H, W, 3] uint8 CUDA tensor in RGB order, 1 <= H, W <= 65500, and returns the
file's bytes.  Buffers are kept for the last frame size and device, as encode_png keeps its own.  There are no quality
or subsampling parameters: cv2's defaults are what save_img writes.
"""
from ._encode import FrameEncoder

MAX_SIDE = 65500

_encoder = FrameEncoder("teco_jpeg", "encode_jpeg")
_state = _encoder.state


def plan_bytes(h, w):
    """(workspace bytes, output capacity) for an h x w frame; ValueError for sizes the encoder does not take."""
    return _encoder.plan_bytes(h, w)


def encode_jpeg(frame_u8):
    """[H, W, 3] uint8 RGB CUDA tensor -> bytes of the JPEG file cv2.imwrite writes for its BGR copy."""
    return _encoder.encode(frame_u8)
