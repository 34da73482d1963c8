"""YUV4MPEG2 (.y4m) streams for `main.py --mode inference --input_y4m / --output_y4m` (DESIGN.md section 4.12).

A Y4M stream is one text header line, `YUV4MPEG2 W<w> H<h> F<n>:<d> I<p> A<n>:<d> C<tag> X<...>`, then frames, each a
`FRAME` line (with optional parameters) followed by the raw 8-bit planes.  Only 4:2:0 limited range is accepted: the
planes are then [3h/2, w] I420 bytes, which cv2.cvtColor(COLOR_YUV2RGB_I420 / COLOR_RGB2YUV_I420) convert -- on the
device here, by kernels.i420_to_rgb and kernels.rgb_to_i420.  The streams are read and written strictly in order,
never seeking, so a FIFO or /dev/stdin (/dev/stdout) works as a path.  This module is host code: the pinned buffers,
the reader thread and the file; the conversions are tecogan_b200/csrc/yuv.cu."""
import collections
import itertools

MAGIC = b'YUV4MPEG2'
MIN_SIDE, MAX_SIDE = 8, 65534         # the engine's smallest input; the conversion kernels' largest side
CHROMA_420 = (None, 'C420', 'C420jpeg', 'C420mpeg2', 'C420paldv')   # one memory layout; the siting is ignored, as cv2 does
HEADER_LIMIT = 4096                   # bytes of a header or FRAME line
PNG_INPUT_RATE, PNG_INPUT_ASPECT = '25:1', '1:1'     # ffmpeg's defaults for an image sequence
READ_RING = 3                         # pinned host frames between the file and the device
READ_CREDITS = 8                      # device frames the reader may hold: frames 0..5 of the warm-up, two ahead

Header = collections.namedtuple('Header', 'w, h, rate, aspect')


def _line(f, what):
    """One '\\n'-terminated line of `f` without its '\\n', b'' at the end of the stream; a line cut short raises."""
    data = f.readline(HEADER_LIMIT + 1)
    if data and not data.endswith(b'\n'):
        raise ValueError('y4m: %s is truncated or longer than %d bytes' % (what, HEADER_LIMIT))
    return data[:-1]


def parse_header(line):
    """The Header of a Y4M stream header line (bytes, without its '\\n').  Refuses, with a ValueError naming the field:
    a wrong magic word, missing or malformed W / H, odd sides or sides outside 8..65534, a C tag other than 4:2:0 8-bit
    (absent, C420, C420jpeg, C420mpeg2, C420paldv), XCOLORRANGE=FULL and interlaced input (It, Ib, Im).  Other X fields
    are ignored; F and A are kept as given (F defaults to 25:1, A to 1:1)."""
    fields = line.split(b' ')
    if fields[0] != MAGIC:
        raise ValueError('y4m: magic word %r is not %r' % (fields[0][:16], MAGIC))
    got = {}
    for raw in fields[1:]:
        if not raw:
            continue
        try:
            tok = raw.decode('ascii')
        except UnicodeDecodeError:
            raise ValueError('y4m: header field %r is not ASCII' % raw[:32])
        tag, val = tok[0], tok[1:]
        if tag == 'X':
            if val.upper() == 'COLORRANGE=FULL':
                raise ValueError('y4m: XCOLORRANGE=FULL: only limited-range 4:2:0 is accepted (write the stream with '
                                 'ffmpeg -pix_fmt yuv420p)')
            continue
        got[tag] = val
    sides = {}
    for tag in 'WH':
        if tag not in got:
            raise ValueError('y4m: header has no %s (frame %s) field' % (tag, 'width' if tag == 'W' else 'height'))
        if not got[tag].isdigit():
            raise ValueError('y4m: field %s%s is not a positive integer' % (tag, got[tag]))
        v = int(got[tag])
        if v % 2 or not MIN_SIDE <= v <= MAX_SIDE:
            raise ValueError('y4m: field %s%d: 4:2:0 sides must be even and %d..%d' % (tag, v, MIN_SIDE, MAX_SIDE))
        sides[tag] = v
    c = got.get('C')
    if (None if c is None else 'C' + c) not in CHROMA_420:
        raise ValueError('y4m: field C%s: only 8-bit 4:2:0 (C420, C420jpeg, C420mpeg2, C420paldv) is accepted; write '
                         'the stream with ffmpeg -pix_fmt yuv420p' % c)
    if got.get('I', 'p') not in ('p', '?'):
        raise ValueError('y4m: field I%s: interlaced input is not accepted, only progressive (Ip)' % got['I'])
    rate, aspect = got.get('F', PNG_INPUT_RATE), got.get('A', PNG_INPUT_ASPECT)
    for tag, val in (('F', rate), ('A', aspect)):
        a, sep, b = val.partition(':')
        if not (sep and a.isdigit() and b.isdigit()):
            raise ValueError('y4m: field %s%s is not <n>:<d>' % (tag, val))
    return Header(sides['W'], sides['H'], rate, aspect)


def format_header(w, h, rate=PNG_INPUT_RATE, aspect=PNG_INPUT_ASPECT):
    """The header line (with its '\\n') this module writes: W, H, F, A, then `Ip C420paldv XCOLORRANGE=LIMITED`."""
    # C420paldv: ffmpeg's y4m demuxer reads it as top-left chroma siting, which is where cv2 takes U and V
    return ('YUV4MPEG2 W%d H%d F%s Ip A%s C420paldv XCOLORRANGE=LIMITED\n' % (w, h, rate, aspect)).encode('ascii')


def frame_bytes(w, h):
    return w * h * 3 // 2


def read_frame(f, out, index):
    """Reads the next frame of `f` into `out` (a writable buffer of frame_bytes) -> False at the end of the stream.  A
    FRAME line that is malformed or a payload cut short raises ValueError naming frame `index` (0-based)."""
    line = _line(f, 'FRAME line of frame %d' % (index + 1))
    if not line:
        return False
    if line != b'FRAME' and not line.startswith(b'FRAME '):
        raise ValueError('y4m: frame %d does not start with FRAME (got %r)' % (index + 1, line[:16]))
    view, got = memoryview(out).cast('B'), 0
    while got < len(view):
        n = f.readinto(view[got:])
        if not n:
            raise ValueError('y4m: frame %d is truncated: %d of %d bytes' % (index + 1, got, len(view)))
        got += n
    return True


class Y4MReader:
    """The inference input from a Y4M stream.  The header is read and checked when the reader is made, before anything
    else is set up.  frames() yields the [h, w, 3] float32 device frames of the stream in the reference's padded order
    (frames 5, 4, 3, 2, 1, then 0, 1, 2, ...; fewer warm-up frames for a stream shorter than 6), each = I420 -> RGB as
    cv2.cvtColor(COLOR_YUV2RGB_I420) gives, then / 255 as the PNG input is (kernels.frames_to_f32).  names() yields the
    names of those frames in the same order, '%04d' of the 1-based frame number; it is consumed in step with frames().
    `limit` > 0 stops after that many frames (--input_dir_len)."""

    def __init__(self, path, limit=-1):
        self.path, self.limit = path, int(limit)
        self.f = open(path, 'rb')
        try:
            head = _line(self.f, 'header')
            if not head:
                raise ValueError('y4m: %s is empty' % path)
            self.header = parse_header(head)
        except BaseException:
            self.f.close()
            raise
        self.warmup = None

    def _chunks(self, scores=False):
        """The reader thread's side: frame k read into a ring of pinned buffers, uploaded and converted on the thread's
        stream; one frame per chunk.  With `scores` each chunk also carries the frame's SAD to the frame before it
        (lib/dataloader.py::scene_sads), computed on the same stream; the previous frame is kept for it."""
        import torch
        from . import kernels as K
        from .lib.dataloader import scene_sads
        w, h = self.header.w, self.header.h
        ring = [torch.empty(frame_bytes(w, h), dtype=torch.uint8, pin_memory=True) for _ in range(READ_RING)]
        copied = [None] * READ_RING
        prev = None
        try:
            for k in (itertools.count() if self.limit <= 0 else range(self.limit)):
                r = k % READ_RING
                if copied[r] is not None:
                    copied[r].synchronize()            # the upload out of this buffer is done
                if not read_frame(self.f, ring[r].numpy(), k):
                    return
                planes = ring[r].to('cuda', non_blocking=True)
                copied[r] = torch.cuda.Event()
                copied[r].record()
                rgb = K.i420_to_rgb(planes.view(3 * h // 2, w))
                if not scores:
                    yield k, [K.frames_to_f32(rgb)[0]]
                    continue
                frame = K.frames_to_f32(rgb)[0]
                sad = scene_sads([frame], prev)
                prev, frame = frame, None
                yield k, [prev], sad
        finally:
            self.f.close()

    def frames(self):
        from .lib.dataloader import DeviceHandoff
        feed = DeviceHandoff(self._chunks(), READ_CREDITS, 'y4m_reader')
        try:
            n0 = 0
            while n0 < 6 and feed.take(n0) is not None:     # the count is unknown: the warm-up needs min(6, n) frames
                n0 += 1
            if n0 == 0:
                return
            self.warmup = min(5, n0 - 1)
            for k in range(self.warmup, 0, -1):             # kept until their second use below
                yield feed.take(k)
            for k in itertools.count():
                frame = feed.take(k)
                if frame is None:
                    return
                feed.drop(k)
                feed.release()
                yield frame
                del frame
        finally:
            feed.close()
            self.f.close()

    def scenes(self, threshold):
        """The stream as lib/dataloader.py::SceneSteps for `main.py --scene_threshold`: scene_order over the cuts where
        score >= threshold, each frame's score computed on the reader's stream.  READ_CREDITS frames cover every scene
        start: its six frames c .. c+5, known before its first step, and two decoded ahead.  name(k) names frame k."""
        from .lib.dataloader import DeviceHandoff, scene_steps
        feed = DeviceHandoff(self._chunks(scores=True), READ_CREDITS, 'y4m_reader')
        try:
            yield from scene_steps(feed, threshold, lambda k: feed.release())
        finally:
            feed.close()
            self.f.close()

    @staticmethod
    def name(k):
        return '%04d' % (k + 1)

    def names(self):
        for k in itertools.chain(range(self.warmup, 0, -1), itertools.count()):
            yield '%04d' % (k + 1)

    def close(self):
        self.f.close()


class Y4MWriter:
    """A Y4M output stream: the header (W, H, F, A of `header`, then Ip C420paldv XCOLORRANGE=LIMITED) when it is
    opened, then one `FRAME` line and the I420 planes per write(), in order.  Errors (a closed FIFO, a full disk) are
    raised: a video with a silently dropped frame is worse than no video."""

    def __init__(self, path, w, h, rate=PNG_INPUT_RATE, aspect=PNG_INPUT_ASPECT):
        if w % 2 or h % 2 or not (2 <= w <= MAX_SIDE and 2 <= h <= MAX_SIDE):
            raise ValueError('y4m: output %dx%d: 4:2:0 sides must be even and 2..%d' % (w, h, MAX_SIDE))
        self.w, self.h = w, h
        self.f = open(path, 'wb')
        try:
            self.f.write(format_header(w, h, rate, aspect))
        except BaseException:
            self.f.close()
            raise

    def write(self, planes):
        """Appends one frame: `planes` holds frame_bytes(w, h) bytes of I420 (a buffer, e.g. a uint8 numpy array)."""
        data = memoryview(planes).cast('B')
        if len(data) != frame_bytes(self.w, self.h):
            raise ValueError('y4m: a %dx%d frame has %d bytes, got %d' % (self.w, self.h, frame_bytes(self.w, self.h),
                                                                          len(data)))
        self.f.write(b'FRAME\n')
        self.f.write(data)

    def close(self):
        self.f.close()
