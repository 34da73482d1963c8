"""The device image encoders' shared host side (tecogan_b200.png, tecogan_b200.jpeg, tecogan_b200.gif): input checks, a
workspace, device output and pinned host buffer kept for the last input size and device, and the two synchronised copies
back."""
import ctypes as C

import torch

from ._ffi import call, lib, ptr, stream_ptr


def check_rgb8(t, name, what, dims):
    """ValueError unless `t` is a contiguous uint8 CUDA tensor of shape [*dims, 3] (dims: a label such as "H, W")."""
    if not torch.is_tensor(t) or t.dtype != torch.uint8:
        raise ValueError("%s: expected a uint8 tensor" % name)
    if not t.is_cuda:
        raise ValueError("%s: the %s must be a CUDA tensor (the encoder has no CPU path)" % (name, what))
    if t.dim() != dims.count(",") + 2 or t.shape[-1] != 3:
        raise ValueError("%s: expected an [%s, 3] RGB %s, got %s" % (name, dims, what, tuple(t.shape)))
    if not t.is_contiguous():
        raise ValueError("%s: the %s must be contiguous" % (name, what))


class FrameEncoder:
    """One C-ABI encoder pair: `<prefix>_plan_bytes(*dims, &ws, &cap)` and
    `<prefix>_encode_rgb8(rgb, *dims, ws, ws_bytes, out, cap, out_len, stream)`, where out_len is a device int64 per
    file (the files lie back to back in out).  PNG and JPEG take dims (H, W), GIF (N, T, H, W)."""

    def __init__(self, prefix, name):
        self.prefix, self.name = prefix, name
        self.state = {}

    def plan_bytes(self, *dims):
        """(workspace bytes, output capacity) for these sizes; ValueError for sizes the encoder does not take."""
        ws, cap = C.c_int64(0), C.c_int64(0)
        call(self.prefix + "_plan_bytes", *[int(d) for d in dims], C.byref(ws), C.byref(cap))
        return ws.value, cap.value

    def _buffers(self, dims, device, nfiles=1):
        st = self.state
        key = (dims, device)
        if st.get("key") != key:
            st.clear()
            ws, cap = self.plan_bytes(*dims)
            st.update(key=key, ws=torch.empty(ws, dtype=torch.uint8, device=device),
                      out=torch.empty(cap, dtype=torch.uint8, device=device),
                      n=torch.empty(nfiles, dtype=torch.int64, device=device),
                      host=torch.empty(cap, dtype=torch.uint8, pin_memory=True),
                      host_n=torch.empty(nfiles, dtype=torch.int64, pin_memory=True))
        return st

    def launch(self, t, dims, nfiles=1):
        """Enqueue the encode of the checked tensor `t` of sizes `dims` and the copy of the file lengths on the current
        stream -> a pending encode for collect().  Until it is collected, this encoder takes no other launch."""
        lib()
        dims = tuple(int(d) for d in dims)
        with torch.cuda.device(t.device):
            b = self._buffers(dims, t.device, nfiles)
            stream = torch.cuda.current_stream()
            call(self.prefix + "_encode_rgb8", ptr(t), *dims, ptr(b["ws"]), b["ws"].numel(), ptr(b["out"]),
                 b["out"].numel(), ptr(b["n"]), stream_ptr())
            b["host_n"].copy_(b["n"], non_blocking=True)
        return b, stream

    def run(self, t, dims, nfiles=1):
        """Encode the checked tensor `t` of sizes `dims` -> the list of its `nfiles` files' bytes."""
        return collect([self.launch(t, dims, nfiles)])[0]

    def encode(self, frame_u8):
        """[H, W, 3] uint8 RGB CUDA tensor -> the file's bytes."""
        check_rgb8(frame_u8, self.name, "frame", "H, W")
        return self.run(frame_u8, frame_u8.shape[:2])[0]


def collect(pending):
    """The files of launched encodes (FrameEncoder.launch), one list per launch: one synchronise for the lengths, the
    byte copies, one synchronise -- however many encodes are pending."""
    for _, stream in pending:
        stream.synchronize()
    lens = [[int(v) for v in b["host_n"].tolist()] for b, _ in pending]
    for (b, stream), ls in zip(pending, lens):
        n = sum(ls)
        with torch.cuda.stream(stream):
            b["host"][:n].copy_(b["out"][:n], non_blocking=True)
    for _, stream in pending:
        stream.synchronize()
    out = []
    for (b, _), ls in zip(pending, lens):
        data = b["host"][:sum(ls)].numpy().tobytes()
        files, o = [], 0
        for k in ls:
            files.append(data[o:o + k])
            o += k
        out.append(files)
    return out
