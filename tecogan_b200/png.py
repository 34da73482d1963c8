"""PNG encoding on the GPU: the bytes cv2.imwrite writes for the same frame (libpng, filter Sub, zlib level 1 with the
run-length strategy), computed by tecogan_b200/csrc/png.cu.  DESIGN.md section 4.5.

encode_png(frame) takes a contiguous [H, W, 3] uint8 CUDA tensor in RGB order and returns the file's bytes.  The
workspace, the device output and the pinned host buffer are kept for the last frame size and device, so a sequence of
equal-sized frames allocates nothing after its first frame.
"""
import ctypes as C

import torch

from ._ffi import call, lib, ptr, stream_ptr

_state = {}


def plan_bytes(h, w):
    """(workspace bytes, output capacity) for an h x w frame; ValueError for sizes the encoder does not take."""
    ws, cap = C.c_int64(0), C.c_int64(0)
    call("teco_png_plan_bytes", int(h), int(w), C.byref(ws), C.byref(cap))
    return ws.value, cap.value


def _buffers(h, w, device):
    key = (h, w, device)
    if _state.get("key") != key:
        _state.clear()
        ws, cap = plan_bytes(h, w)
        _state.update(key=key, ws=torch.empty(ws, dtype=torch.uint8, device=device),
                      out=torch.empty(cap, dtype=torch.uint8, device=device),
                      n=torch.empty(1, dtype=torch.int64, device=device),
                      host=torch.empty(cap, dtype=torch.uint8, pin_memory=True),
                      host_n=torch.empty(1, dtype=torch.int64, pin_memory=True))
    return _state


def encode_png(frame_u8):
    """[H, W, 3] uint8 RGB CUDA tensor -> bytes of the PNG file cv2.imwrite writes for its BGR copy."""
    t = frame_u8
    if not torch.is_tensor(t) or t.dtype != torch.uint8:
        raise ValueError("encode_png: expected a uint8 tensor")
    if not t.is_cuda:
        raise ValueError("encode_png: the frame must be a CUDA tensor (the encoder has no CPU path)")
    if t.dim() != 3 or t.shape[2] != 3:
        raise ValueError("encode_png: expected an [H, W, 3] RGB frame, got %s" % (tuple(t.shape),))
    if not t.is_contiguous():
        raise ValueError("encode_png: the frame must be contiguous")
    lib()
    h, w = int(t.shape[0]), int(t.shape[1])
    with torch.cuda.device(t.device):
        b = _buffers(h, w, t.device)
        stream = torch.cuda.current_stream()
        call("teco_png_encode_rgb8", ptr(t), h, w, ptr(b["ws"]), b["ws"].numel(), ptr(b["out"]), b["out"].numel(),
             ptr(b["n"]), stream_ptr())
        b["host_n"].copy_(b["n"], non_blocking=True)
        stream.synchronize()
        n = int(b["host_n"][0])
        b["host"][:n].copy_(b["out"][:n], non_blocking=True)
        stream.synchronize()
        return b["host"][:n].numpy().tobytes()
