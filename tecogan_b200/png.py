"""PNG encoding and decoding on the GPU.

encode_png(frame) takes a contiguous [H, W, 3] uint8 CUDA tensor in RGB order and returns the bytes cv2.imwrite writes
for the same frame (libpng, filter Sub, zlib level 1 with the run-length strategy), computed by
tecogan_b200/csrc/png.cu (DESIGN.md section 4.5).  The workspace, the device output and the pinned host buffer are kept
for the last frame size and device, so a sequence of equal-sized frames allocates nothing after its first frame.

decode_png(paths) and decode_png_into(paths, buf, offsets, sizes) give the pixels cv2.imread(path, IMREAD_COLOR)[..., ::-1]
gives, as uint8 RGB on the device (tecogan_b200/csrc/png_decode.cu, DESIGN.md section 4.7).  The host reads each file,
walks its chunks and checks every CRC; a file inside the subset the device takes has its zlib stream decoded there, and
every other file -- or one whose stream the device reports as anything but exact -- is decoded by cv2 on the host.
"""
import concurrent.futures
import ctypes as C
import struct
import zlib

import numpy as np
import torch

from ._encode import FrameEncoder
from ._ffi import call, ptr, stream_ptr

_encoder = FrameEncoder("teco_png", "encode_png")
_state = _encoder.state


def plan_bytes(h, w):
    """(workspace bytes, output capacity) for an h x w frame; ValueError for sizes the encoder does not take."""
    return _encoder.plan_bytes(h, w)


def encode_png(frame_u8):
    """[H, W, 3] uint8 RGB CUDA tensor -> bytes of the PNG file cv2.imwrite writes for its BGR copy."""
    return _encoder.encode(frame_u8)


# ------------------------------------------------------------------------------------------------ decoding
SIGNATURE = b"\x89PNG\r\n\x1a\n"
MAX_DIM = 65500
MAX_PIXELS = 1 << 30                                 # cv2.imread refuses larger frames (CV_IO_MAX_IMAGE_PIXELS)
DEPTHS = {0: (1, 2, 4, 8), 2: (8,), 3: (1, 2, 4, 8), 4: (8,), 6: (8,)}   # colour type -> bit depths the device takes
REFUSED = (b"eXIf", b"acTL", b"fcTL", b"fdAT")      # eXIf turns cv2's frame; APNG chunks: cv2 reads those on its own
DESC_COLS = 11
BATCH_BYTES = 256 << 20
# teco_png_decode_rgb8's per-file status (include/teco.h); anything but OK sends the file to cv2
STATUS = {0: "ok", 1: "zlib header", 2: "block type or stored length", 3: "Huffman code", 4: "symbol outside the code",
          5: "distance out of range", 6: "stream ends early", 7: "too many bytes", 8: "too few bytes", 9: "Adler-32",
          10: "data after the stream", 11: "filter type", 12: "palette index", 13: "descriptor"}


class Stream:
    """What the device needs of one file: IHDR's size and format, the concatenated IDAT data and the PLTE bytes."""
    __slots__ = ("h", "w", "colour", "depth", "idat", "plte")

    def __init__(self, h, w, colour, depth, idat, plte):
        self.h, self.w, self.colour, self.depth, self.idat, self.plte = h, w, colour, depth, idat, plte


def parse_png(data):
    """The chunk walk: a Stream when the file is inside the subset the device decodes (DESIGN.md section 4.7), None
    when cv2 has to decode it -- no PNG signature, a chunk past the end of the file or with a bad CRC, 16-bit or
    interlaced or an unknown format, a side above 65 500 or more than 2^30 pixels (cv2 raises there), eXIf or APNG chunks, an unknown critical chunk, IDAT chunks
    that are not consecutive, a missing or misplaced PLTE, anything after IEND.  Only CRCs and the chunk order are
    checked here; whether the zlib stream decodes exactly is known after the device has decoded it."""
    mv = memoryview(data)
    if bytes(mv[:8]) != SIGNATURE:
        return None
    pos, n = 8, len(data)
    ihdr, plte, idat = None, None, []
    idat_state = 0                                   # 0: no IDAT yet, 1: in the IDAT run, 2: after it
    while True:
        if pos + 12 > n:
            return None
        length = struct.unpack_from(">I", data, pos)[0]
        kind = bytes(mv[pos + 4:pos + 8])
        if length > 0x7FFFFFFF or pos + 12 + length > n or not kind.isalpha():
            return None
        body = mv[pos + 8:pos + 8 + length]
        if zlib.crc32(body, zlib.crc32(kind)) != struct.unpack_from(">I", data, pos + 8 + length)[0]:
            return None
        pos += 12 + length
        if ihdr is None:
            if kind != b"IHDR" or length != 13:
                return None
            w, h, depth, colour, comp, filt, interlace = struct.unpack(">IIBBBBB", body)
            if not (1 <= h <= MAX_DIM and 1 <= w <= MAX_DIM) or h * w > MAX_PIXELS or depth not in DEPTHS.get(colour, ()) \
                    or comp or filt or interlace:
                return None
            ihdr = (h, w, colour, depth)
            continue
        if kind == b"IDAT":
            if idat_state == 2:
                return None
            idat_state = 1
            idat.append(body)
            continue
        if idat_state == 1:
            idat_state = 2
        if kind == b"IEND":
            if length or pos != n:
                return None
            break
        if kind == b"PLTE":
            if plte is not None or idat_state or ihdr[2] in (0, 4) or length % 3 or not 3 <= length <= 768:
                return None
            plte = body
            continue
        if kind in REFUSED or kind == b"IHDR" or not kind[0] & 0x20:     # bit 5 clear in the first letter: critical
            return None
    h, w, colour, depth = ihdr
    if not idat or (colour == 3 and plte is None):
        return None
    return Stream(h, w, colour, depth, b"".join(idat), bytes(plte) if colour == 3 else b"")


def load_png(path):
    """parse_png of the file at `path`."""
    with open(path, "rb") as f:
        return parse_png(f.read())


def imread_rgb(path):
    """cv2.imread(path, IMREAD_COLOR) as contiguous RGB; ValueError when cv2 cannot decode the file."""
    import cv2
    im = cv2.imread(path, cv2.IMREAD_COLOR)
    if im is None:
        raise ValueError("cannot decode " + path)
    return np.ascontiguousarray(im[:, :, ::-1])


def decode_plan_bytes(h, w, colour, depth):
    """Workspace bytes the device decoder needs for one file of this size and format."""
    ws = C.c_int64(0)
    call("teco_png_decode_plan_bytes", int(h), int(w), int(colour), int(depth), C.byref(ws))
    return ws.value


def decode_streams(items, dst, pool=None, batch_bytes=BATCH_BYTES):
    """items: [(Stream, byte offset in dst)].  Decodes each stream into the flat uint8 CUDA tensor `dst` as a packed
    [h, w, 3] frame at its offset, in batches of at most `batch_bytes` of workspace (one file may exceed it alone), and
    returns the int32 status of every item (0: decoded; otherwise its bytes in dst are undefined)."""
    if not (torch.is_tensor(dst) and dst.is_cuda and dst.dtype == torch.uint8 and dst.dim() == 1 and dst.is_contiguous()):
        raise ValueError("decode_streams: dst must be a flat contiguous uint8 CUDA tensor")
    out = np.zeros(len(items), np.int32)
    ws_need = [decode_plan_bytes(s.h, s.w, s.colour, s.depth) for s, _ in items]
    for s, off in items:
        if off < 0 or off + s.h * s.w * 3 > dst.numel():
            raise ValueError("decode_streams: a %dx%d frame at byte %d does not fit in %d bytes" % (s.h, s.w, off, dst.numel()))
    with torch.cuda.device(dst.device):
        for i, j in _windows(ws_need, batch_bytes):
            out[i:j] = _decode_batch(items[i:j], ws_need[i:j], sum(ws_need[i:j]), dst, pool)
    return out


def _decode_batch(items, ws_need, ws_total, dst, pool):
    args = stage_batch(items, ws_need, ws_total, dst, pool)
    launch_batch(*args)
    return args[-1].cpu().numpy()


def stage_batch(items, ws_need, ws_total, dst, pool=None):
    """The inputs of one teco_png_decode_rgb8 launch on dst's device: the packed streams and palettes, the
    descriptors, the workspace and the status array (copies queued on the current stream)."""
    n = len(items)
    desc = np.zeros((n, DESC_COLS), np.int64)
    src_off = ws_off = 0
    for k, (s, off) in enumerate(items):
        zl = len(s.idat)
        desc[k] = (src_off, zl, s.h, s.w, s.colour, s.depth, src_off + zl, len(s.plte) // 3, off, 3 * s.w, ws_off)
        src_off += zl + len(s.plte)
        ws_off += ws_need[k]
    stage = torch.empty(max(1, src_off), dtype=torch.uint8, pin_memory=True)
    host = stage.numpy()

    def pack(k):
        s, a = items[k][0], int(desc[k, 0])
        host[a:a + len(s.idat)] = np.frombuffer(s.idat, np.uint8)
        host[a + len(s.idat):a + len(s.idat) + len(s.plte)] = np.frombuffer(s.plte, np.uint8)
    list(pool.map(pack, range(n)) if pool is not None else map(pack, range(n)))
    dev = dst.device
    src = stage.to(dev, non_blocking=True)
    d = torch.from_numpy(desc).pin_memory().to(dev, non_blocking=True)
    ws = torch.empty(max(1, ws_total), dtype=torch.uint8, device=dev)
    status = torch.empty(n, dtype=torch.int32, device=dev)
    return src, d, ws, dst, status


def launch_batch(src, desc, ws, dst, status):
    """The three kernels of one batch staged by stage_batch, on the current stream."""
    call("teco_png_decode_rgb8", ptr(src), src.numel(), ptr(desc), desc.shape[0], ptr(ws), ws.numel(), ptr(dst),
         dst.numel(), ptr(status), stream_ptr())


def _windows(costs, budget):
    """Consecutive [i, j) ranges whose costs sum to at most `budget` (a single item may exceed it)."""
    i = 0
    while i < len(costs):
        j, total = i + 1, costs[i]
        while j < len(costs) and total + costs[j] <= budget:
            total += costs[j]
            j += 1
        yield i, j
        i = j


# Rates measured on an H100 80GB HBM3 (700 W) host (DESIGN.md section 7): one warp inflates about 5 MB of filtered bytes
# per second whatever the frame size, one cv2.imread thread decodes up to 85 MB of RGB per second.
WARP_BYTES_PER_S = 5.0e6
CV2_BYTES_PER_S = 85.0e6
SLACK_S = 0.05


def device_pays(sizes, threads, batch_bytes=BATCH_BYTES):
    """Whether the device is expected to decode frames of these (h, w) sizes (one window) faster than `threads` cv2
    threads would.  Files in one batch inflate side by side, so a batch takes about as long as its largest file, while
    cv2 takes the total spread over its threads: the device wins with many files per batch and loses with few large
    ones (a handful of 4K frames, a store of 1080p frames against six threads).  Within SLACK_S the device is kept.
    Sizes come from the IHDR chunks, so the choice is made before anything is read beyond them."""
    if not len(sizes):
        return False
    ws = [int(h) * (3 * int(w) + 1) for h, w in sizes]           # filtered bytes of an RGB frame
    t_dev = sum(max(ws[i:j]) for i, j in _windows(ws, batch_bytes)) / WARP_BYTES_PER_S
    t_host = sum(int(h) * int(w) * 3 for h, w in sizes) / (max(1, int(threads)) * CV2_BYTES_PER_S)
    return t_dev <= t_host + SLACK_S


def png_size(path):
    """(h, w) from the file's IHDR, or None when it does not start like a PNG."""
    with open(path, "rb") as f:
        head = f.read(24)
    if len(head) == 24 and head[:8] == SIGNATURE and head[12:16] == b"IHDR":
        w, h = struct.unpack(">II", head[16:24])
        return int(h), int(w)
    return None


def _host_into(ks, paths, buf, offsets, sizes, pool, host_decode):
    """Files ks decoded by host_decode on the pool into a pinned stage, then copied into their slots of buf."""
    if not ks:
        return
    n = [int(sizes[k, 0] * sizes[k, 1] * 3) for k in ks]
    at = np.concatenate([[0], np.cumsum(n)]).astype(np.int64)
    stage = torch.empty(max(1, int(at[-1])), dtype=torch.uint8, pin_memory=True)
    hs = stage.numpy()

    def put(q):
        k = ks[q]
        im = host_decode(paths[k])
        h, w = int(sizes[k, 0]), int(sizes[k, 1])
        if tuple(im.shape) != (h, w, 3):
            raise ValueError("%s decodes to %s, its slot holds %dx%d" % (paths[k], tuple(im.shape), h, w))
        hs[at[q]:at[q + 1]] = np.ascontiguousarray(im).reshape(-1)
    list(pool.map(put, range(len(ks))))
    with torch.cuda.device(buf.device):
        for q, k in enumerate(ks):
            buf[int(offsets[k]):int(offsets[k]) + n[q]].copy_(stage[int(at[q]):int(at[q + 1])], non_blocking=True)
        torch.cuda.current_stream().synchronize()            # the stage is freed on return


def decode_png_into(paths, buf, offsets, sizes, threads=1, batch_bytes=BATCH_BYTES, host_decode=imread_rgb):
    """Decodes file k of `paths` into the flat uint8 CUDA tensor `buf` as a packed [h, w, 3] RGB frame at byte
    offsets[k], sizes[k] = (h, w): the pixels cv2.imread gives.  Host threads read the files, walk their chunks and pack
    the compressed streams; the device decodes them, `batch_bytes` of frames at a time, unless device_pays expects
    cv2 on `threads` threads to be faster for that window (then all its files go to `host_decode`).  Files outside the
    device's subset, and files whose stream the device reports as inexact, are decoded by `host_decode(path)` (an [h, w, 3] RGB
    array) and copied into their slot.  A file that decodes to another size than sizes[k] raises ValueError."""
    offsets = np.asarray(offsets, np.int64)
    sizes = np.asarray(sizes, np.int64).reshape(-1, 2)
    if not (len(paths) == len(offsets) == len(sizes)):
        raise ValueError("decode_png_into: %d paths, %d offsets, %d sizes" % (len(paths), len(offsets), len(sizes)))
    nbytes = sizes[:, 0] * sizes[:, 1] * 3
    windows = [(i, j, device_pays(sizes[i:j], threads, batch_bytes)) for i, j in _windows(nbytes.tolist(), batch_bytes)]
    with concurrent.futures.ThreadPoolExecutor(max_workers=max(1, int(threads))) as pool:
        def read(w):
            i, j, on_dev = windows[w]
            return pool.map(load_png, paths[i:j]) if on_dev else None
        reads = read(0) if windows else None
        for w, (i, j, on_dev) in enumerate(windows):
            if not on_dev:
                _host_into(list(range(i, j)), paths, buf, offsets, sizes, pool, host_decode)
                reads = read(w + 1) if w + 1 < len(windows) else None
                continue
            streams = list(reads)
            if w + 1 < len(windows):        # the next window's files are read while the device decodes this one
                reads = read(w + 1)
            dev = [k for k in range(i, j) if streams[k - i] is not None]
            for k in dev:
                s = streams[k - i]
                if (s.h, s.w) != tuple(sizes[k]):
                    raise ValueError("%s decodes to %dx%d, its slot holds %dx%d" % (paths[k], s.h, s.w, *sizes[k]))
            status = decode_streams([(streams[k - i], int(offsets[k])) for k in dev], buf, None, batch_bytes)
            host = [k for k in range(i, j) if streams[k - i] is None] + [k for k, st in zip(dev, status) if st]
            _host_into(host, paths, buf, offsets, sizes, pool, host_decode)


def decode_png(paths, device=None, threads=1, batch_bytes=BATCH_BYTES, host_decode=imread_rgb):
    """[H, W, 3] uint8 RGB CUDA tensors of the files at `paths`, in order: the pixels cv2.imread gives.  Files are read
    in windows of at most `batch_bytes` on disk and decoded on the device as decode_png_into does (device_pays chooses
    per window); files outside the device's subset or with an inexact stream come from `host_decode(path)`.  The frames of one window are views of one
    device buffer."""
    device = torch.device("cuda") if device is None else torch.device(device)
    if device.type != "cuda":
        raise ValueError("decode_png: the frames are decoded on a CUDA device, got %s" % device)
    import os
    out = [None] * len(paths)
    with concurrent.futures.ThreadPoolExecutor(max_workers=max(1, int(threads))) as pool:
        hw = list(pool.map(png_size, paths))
        for i, j in _windows([os.path.getsize(p) for p in paths], batch_bytes):
            if not device_pays([x for x in hw[i:j] if x], threads, batch_bytes):
                for k, im in zip(range(i, j), pool.map(host_decode, paths[i:j])):
                    out[k] = torch.from_numpy(np.ascontiguousarray(im)).to(device)
                continue
            streams = list(pool.map(load_png, paths[i:j]))
            dev = [k for k in range(i, j) if streams[k - i] is not None]
            offs = np.concatenate([[0], np.cumsum([streams[k - i].h * streams[k - i].w * 3 for k in dev])]).astype(np.int64)
            flat = torch.empty(max(1, int(offs[-1])), dtype=torch.uint8, device=device)
            status = decode_streams([(streams[k - i], int(o)) for k, o in zip(dev, offs)], flat, pool, batch_bytes)
            host = [k for k in range(i, j) if streams[k - i] is None]
            for k, o, st in zip(dev, offs, status):
                s = streams[k - i]
                if st:
                    host.append(k)
                else:
                    out[k] = flat[int(o):int(o) + s.h * s.w * 3].view(s.h, s.w, 3)
            for k, im in zip(host, pool.map(host_decode, [paths[k] for k in host])):
                out[k] = torch.from_numpy(np.ascontiguousarray(im)).to(device)
    return out
