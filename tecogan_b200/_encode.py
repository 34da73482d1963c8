"""The device image encoders' shared host side (tecogan_b200.png, tecogan_b200.jpeg): input checks, a workspace, device
output and pinned host buffer kept for the last frame size and device, and the two synchronised copies back."""
import ctypes as C

import torch

from ._ffi import call, lib, ptr, stream_ptr


class FrameEncoder:
    """One C-ABI encoder pair: `<prefix>_plan_bytes(H, W, &ws, &cap)` and
    `<prefix>_encode_rgb8(rgb, H, W, ws, ws_bytes, out, cap, out_len, stream)`."""

    def __init__(self, prefix, name):
        self.prefix, self.name = prefix, name
        self.state = {}

    def plan_bytes(self, h, w):
        """(workspace bytes, output capacity) for an h x w frame; ValueError for sizes the encoder does not take."""
        ws, cap = C.c_int64(0), C.c_int64(0)
        call(self.prefix + "_plan_bytes", int(h), int(w), C.byref(ws), C.byref(cap))
        return ws.value, cap.value

    def _buffers(self, h, w, device):
        st = self.state
        key = (h, w, device)
        if st.get("key") != key:
            st.clear()
            ws, cap = self.plan_bytes(h, w)
            st.update(key=key, ws=torch.empty(ws, dtype=torch.uint8, device=device),
                      out=torch.empty(cap, dtype=torch.uint8, device=device),
                      n=torch.empty(1, dtype=torch.int64, device=device),
                      host=torch.empty(cap, dtype=torch.uint8, pin_memory=True),
                      host_n=torch.empty(1, dtype=torch.int64, pin_memory=True))
        return st

    def encode(self, frame_u8):
        """[H, W, 3] uint8 RGB CUDA tensor -> the file's bytes."""
        t, name = frame_u8, self.name
        if not torch.is_tensor(t) or t.dtype != torch.uint8:
            raise ValueError("%s: expected a uint8 tensor" % name)
        if not t.is_cuda:
            raise ValueError("%s: the frame must be a CUDA tensor (the encoder has no CPU path)" % name)
        if t.dim() != 3 or t.shape[2] != 3:
            raise ValueError("%s: expected an [H, W, 3] RGB frame, got %s" % (name, tuple(t.shape)))
        if not t.is_contiguous():
            raise ValueError("%s: the frame must be contiguous" % name)
        lib()
        h, w = int(t.shape[0]), int(t.shape[1])
        with torch.cuda.device(t.device):
            b = self._buffers(h, w, t.device)
            stream = torch.cuda.current_stream()
            call(self.prefix + "_encode_rgb8", ptr(t), h, w, ptr(b["ws"]), b["ws"].numel(), ptr(b["out"]),
                 b["out"].numel(), ptr(b["n"]), stream_ptr())
            b["host_n"].copy_(b["n"], non_blocking=True)
            stream.synchronize()
            n = int(b["host_n"][0])
            b["host"][:n].copy_(b["out"][:n], non_blocking=True)
            stream.synchronize()
            return b["host"][:n].numpy().tobytes()
