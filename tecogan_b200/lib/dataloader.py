"""Mirror of the reference's lib/dataloader.py: the inference PNG loader (lib/dataloader.py:11-50), the device half of
frvsr_gpu_data_loader (lib/dataloader.py:306-332) and -- as the caller side of the training path -- a host loader for
HR training clips (`HRClipLoader`) that follows `loadHR` + `tf.train.shuffle_batch` (lib/dataloader.py:147-273): same
directory layout, frame windows, moving-first-frame / random-crop / flip augmentation, a thread pool instead of TF queue
runners.  The validation split (lib/dataloader.py:287-296) is a second `HRClipLoader` over the held-out scenes
(`validation_loader`); it feeds the val_* summaries of main.py --mode train --summary_dir.  `FrameStore` is the device
half: the frames of those scenes decoded once into device memory (or into host memory mapped into the device's address
space), the same batches cut there by teco_gather_clips_u8 (teco_gather_clips_host_u8)."""
import collections
import concurrent.futures
import itertools
import math
import os
import struct
import time

import numpy as np

from .. import kernels as K
from .ops import preprocess


INFERENCE_THREADS = max(1, min(8, os.cpu_count() or 1))


def inference_paths(FLAGS):
    """The files of the inference input (reference lib/dataloader.py:11-36) -> (paths, down): the .png files of
    --input_dir_LR, or of --input_dir_HR when the LR directory is not given or missing (down = True: those frames are
    down-sampled), sorted by the digits of their names and cut to --input_dir_len when it is positive."""
    filedir = FLAGS.input_dir_LR
    downSP = False
    if (FLAGS.input_dir_LR is None) or (not os.path.exists(FLAGS.input_dir_LR)):
        if (FLAGS.input_dir_HR is None) or (not os.path.exists(FLAGS.input_dir_HR)):
            raise ValueError('Input directory not found')
        filedir = FLAGS.input_dir_HR
        downSP = True
    names = [_ for _ in os.listdir(filedir) if _.endswith(".png")]
    names = sorted(names)
    names.sort(key=lambda f: int(''.join(list(filter(str.isdigit, f))) or -1))
    if FLAGS.input_dir_len > 0:
        names = names[:FLAGS.input_dir_len]
    return [os.path.join(filedir, _) for _ in names], downSP


def padded(seq):
    """The reference's hard-coded symmetric warm-up padding: entries 5, 4, 3, 2, 1 prepended (fewer for a shorter
    sequence)."""
    return seq[5:0:-1] + seq


def scene_threshold(value):
    """The threshold T of --scene_threshold as a float: 0 < T <= 100 and finite, else ValueError (also for a value that
    is not a number)."""
    try:
        t = float(value)
    except (TypeError, ValueError):
        raise ValueError('--scene_threshold: %r is not a number' % (value,))
    if not (math.isfinite(t) and 0.0 < t <= 100.0):
        raise ValueError('--scene_threshold must be in (0, 100], got %r' % (value,))
    return t


def scene_score(sad, values, prev_mafd):
    """(mafd, score) of a frame whose 8-bit difference to the previous frame sums to `sad` over `values` values (3 h w):
    mafd = 100 sad / (255 values), the mean absolute frame difference on a 0..100 scale, and score = min(mafd,
    |mafd - prev_mafd|), so that a sustained fast pan is not a cut.  Float64; a scene starts where score >= T."""
    mafd = 100.0 * sad / (values * 255.0)
    return mafd, min(mafd, abs(mafd - prev_mafd))


def scene_order(cuts):
    """The inference order of a stream cut into scenes, built as the stream arrives.  `cuts` yields (index, cut) in
    stream order (index 0, 1, 2, ...; cut: a scene starts at that frame; frame 0 always starts one).  Yields
    (input index, write, reset before) steps: each scene of L frames starting at frame c is run as the reference runs a
    sequence (padded): warm-up frames c+m, ..., c+1 (not written), m = min(5, L - 1), then c, ..., c+L-1 (each written
    once), with the recurrence reset before the scene's first step.  Without a cut and with n >= 6 frames this is
    padded(range(n)) with writes from position 5.

    `cuts` is read lazily: at most six pairs past a scene's first frame (enough to bound m) and, inside a scene, one
    pair past the step last yielded (to know whether the next frame starts a scene)."""
    it = iter(cuts)
    ahead = collections.deque()                  # pairs read but not yet placed

    def have(count):
        while len(ahead) < count:
            got = next(it, None)
            if got is None:
                return False
            ahead.append(got)
        return True
    while have(1):
        c = ahead.popleft()[0]                   # a scene starts here
        extent = 1                               # the scene's frames within c .. c+5
        while extent < 6 and have(extent) and not ahead[extent - 1][1]:
            extent += 1
        m = extent - 1
        for k in range(c + m, c, -1):
            yield k, False, k == c + m
        yield c, True, m == 0
        while have(1) and not ahead[0][1]:
            yield ahead.popleft()[0], True, False


def inference_data_loader(FLAGS):
    """reference lib/dataloader.py:11-50: sorted PNG list -> RGB float32 /255 frames, with the hard-coded symmetric
    warm-up padding (list indices 5,4,3,2,1 prepended).  inputs[k] is an [h, w, 3] float32 CUDA tensor (read_inputs);
    the padding entries are the same tensors as the frames they repeat.  The whole sequence stays on the device;
    stream_inputs gives the same frames holding about two windows of them at a time."""
    image_list_LR, downSP = inference_paths(FLAGS)
    image_LR = read_inputs(image_list_LR, downSP)
    Data = collections.namedtuple('Data', 'paths_LR, inputs')
    return Data(paths_LR=padded(image_list_LR), inputs=padded(image_LR))


def input_windows(paths, window_bytes=None):
    """The [i, j) windows stream_inputs decodes `paths` in: consecutive files whose decoded input (8- or 16-bit RGB from
    the PNG header, the file size for a file that is not a PNG) sums to at most `window_bytes` (png.BATCH_BYTES by
    default); a single larger file is a window of its own."""
    from .. import png
    budget = png.BATCH_BYTES if window_bytes is None else int(window_bytes)
    return list(png._windows([_input_cost(p) for p in paths], budget))


def _input_cost(path):
    hd = _png_head(path)
    return hd[0] * hd[1] * 3 * (2 if hd[2] > 8 else 1) if hd else os.path.getsize(path)


def stream_inputs(paths, down, window_bytes=None):
    """Generator over the frames inference_data_loader(...).inputs holds, in the same padded order
    (padded(paths) = paths[5:0:-1] + paths), without keeping the sequence on the device.

    A reader thread decodes the files window by window (input_windows) with read_inputs(window_paths, down) on a CUDA
    stream of its own, one window ahead of the consumer (DeviceHandoff).  Each file is decoded once: the warm-up entries
    are the same tensors as frames 1..5, which are kept until the sequence passes them again.  A decoding error is raised
    by the generator at the frame that needs the window.  Closing the generator (or an exception in it) stops and joins
    the reader."""
    windows = input_windows(paths, window_bytes)
    if not windows:
        return
    n = len(paths)
    order = padded(list(range(n)))
    last_use = {k: p for p, k in enumerate(order)}
    window_of = [w for w, (i, j) in enumerate(windows) for _ in range(i, j)]
    left = [j - i for i, j in windows]              # files of each window not yet past their last use
    # the warm-up needs every window up to file min(5, n - 1), window w5, before its first frame, and one more may be
    # decoded ahead; the windows before w5 return no credit, so past the warm-up the reader is one window ahead
    w5 = window_of[order[0]]

    def decode():
        for i, j in windows:
            yield i, list(read_inputs(paths[i:j], down))

    feed = DeviceHandoff(decode(), w5 + 2, 'stream_inputs')
    try:
        for p, k in enumerate(order):
            frame = feed.take(k)
            if last_use[k] == p:
                feed.drop(k)
                w = window_of[k]
                left[w] -= 1
                if left[w] == 0 and w >= w5:
                    feed.release()
            yield frame
            del frame
    finally:
        feed.close()


# One step of a stream cut into scenes: the [h, w, 3] float32 frame, its input index, whether it is written (False: a
# warm-up step), whether the recurrence is reset before it and, on a scene's first step, the scene's first frame and the
# score that started it (None for the stream's first scene).
SceneStep = collections.namedtuple('SceneStep', 'frame, index, write, reset, start, score')


def scene_steps(feed, threshold, release):
    """The steps of a stream cut into scenes (scene_order), its frames taken from `feed` (a DeviceHandoff whose chunks
    carry each frame's 8-bit SAD to the previous frame, frame_sad_q8, in pinned memory) in stream order.  A frame's score
    is read on the host after a wait on the reader's event for its chunk (DeviceHandoff.value), never on the consumer's
    stream.  A frame is dropped once its written step has been handed out, then release(k) is called."""
    cut_at = collections.deque()                 # (frame, score) of the cuts found and not yet reached

    def cuts():
        prev_mafd = 0.0
        for k in itertools.count():
            frame = feed.take(k)
            if frame is None:
                return
            if k == 0:
                yield 0, True
                continue
            prev_mafd, score = scene_score(feed.value(k), frame.numel(), prev_mafd)
            del frame
            if score >= threshold:
                cut_at.append((k, score))
            yield k, score >= threshold
    first = True
    for k, write, reset in scene_order(cuts()):
        start = score = None
        if reset:
            start, score = (0, None) if first else cut_at.popleft()
            first = False
        frame = feed.take(k)
        yield SceneStep(frame, k, write, reset, start, score)
        del frame
        if write:
            feed.drop(k)
            release(k)


def scene_sads(frames, prev):
    """The reader side of scene_steps: a pinned int64 tensor with frame_sad_q8 of each of `frames` against the frame
    before it (`prev` for the first, 0 without one or for a frame of another size), copied on the current stream."""
    import torch
    sad = torch.zeros(len(frames), dtype=torch.int64, device=frames[0].device)
    for t, f in enumerate(frames):
        if prev is not None and prev.shape == f.shape:
            K.frame_sad_q8(prev, f, sad[t:t + 1])
        prev = f
    host = torch.empty(len(frames), dtype=torch.int64, pin_memory=True)
    host.copy_(sad, non_blocking=True)
    return host


def stream_scenes(paths, down, threshold, window_bytes=None):
    """Generator over the SceneSteps of the PNG input of `main.py --scene_threshold T`: the frames of stream_inputs,
    decoded the same way, in the order scene_order gives for the cuts where score >= T.

    The reader thread computes each frame's SAD to the frame before it on its own stream, right after the window is
    decoded (scene_sads; it keeps a reference to the window's last frame for the next window).  A window returns its
    credit once every frame of it has been written.  The credits are the most windows any frames c .. c+5 span, plus
    one to decode ahead: at a scene's first frame c every earlier window has returned its credit, and the scene's extent
    within c .. c+5 must be known before its first step.  So the frames on the device stay bounded by that, whatever
    the stream's length or number of cuts.  Errors, closing and the reader thread are as in stream_inputs."""
    windows = input_windows(paths, window_bytes)
    if not windows:
        return
    n = len(paths)
    window_of = [w for w, (i, j) in enumerate(windows) for _ in range(i, j)]
    left = [j - i for i, j in windows]
    credits = max(window_of[min(c + 5, n - 1)] - window_of[c] + 1 for c in range(n)) + 1

    def decode():
        prev = None
        for i, j in windows:
            frames = list(read_inputs(paths[i:j], down))
            yield i, frames, scene_sads(frames, prev)
            prev = frames[-1]
            del frames

    def release(k):
        w = window_of[k]
        left[w] -= 1
        if left[w] == 0:
            feed.release()
    feed = DeviceHandoff(decode(), credits, 'stream_scenes')
    try:
        yield from scene_steps(feed, threshold, release)
    finally:
        feed.close()


class DeviceHandoff:
    """The reader half of a streamed inference input, shared by stream_inputs (PNG files) and
    tecogan_b200/y4m.py::Y4MReader (a YUV4MPEG2 stream).

    A reader thread runs `chunks` -- an iterator of (first frame index, [frames]) -- under a CUDA stream of its own, one
    credit per chunk: it waits for a credit before it asks for the next chunk, and the consumer gives credits back with
    release().  Each chunk is handed over with an event recorded on the reader's stream.  take(k) returns frame k: the
    consumer's current stream first waits for the chunk's event, and the chunk's tensors are recorded on that stream, so
    the allocator reuses their memory only once the consumer's work on them is done.  take() returns None once the
    iterator has ended without frame k, and raises an exception of the reader at the frame that needs its chunk.  drop(k)
    forgets frame k.  close() stops and joins the reader; the iterator is not asked for another chunk after it.

    A chunk may carry a third item, a host tensor with one value per frame written on the reader's stream (the scene
    scores' pinned SADs, scene_sads): value(k) returns frame k's entry after a host wait on the chunk's event alone, so
    the consumer's stream is never synchronised to read it."""

    def __init__(self, chunks, credits, name):
        import queue
        import threading
        import torch
        self.credits, self.ready, self.stop = threading.Semaphore(credits), queue.Queue(), threading.Event()
        self.have, self.values, self.ended = {}, {}, False
        cuda = torch.cuda.is_available()
        device = torch.cuda.current_device() if cuda else None

        def read():
            try:
                if cuda:
                    torch.cuda.set_device(device)
                stream = torch.cuda.Stream() if cuda else None
                it = iter(chunks)
                while True:
                    self.credits.acquire()
                    if self.stop.is_set():
                        return
                    with torch.cuda.stream(stream):
                        got = next(it, None)
                        if got is None:
                            self.ready.put(None)
                            return
                        i, frames = got[:2]
                        done = torch.cuda.Event() if cuda else None
                        if cuda:
                            done.record()
                    self.ready.put((i, frames, done) + tuple(got[2:]))
                    del got, frames
            except BaseException as e:              # handed to the consumer, raised there
                self.ready.put(e)
            finally:
                close = getattr(chunks, 'close', None)
                if close is not None:               # a generator's own clean-up runs on this thread
                    close()

        self.thread = threading.Thread(target=read, name=name, daemon=True)
        self.thread.start()

    def take(self, k):
        import torch
        while k not in self.have:
            if self.ended:
                return None
            got = self.ready.get()
            if got is None:
                self.ended = True
                continue
            if isinstance(got, BaseException):
                self.ended = True
                raise got
            i, frames, done = got[:3]
            if len(got) > 3:
                self.values.update((i + t, (done, got[3], t)) for t in range(len(frames)))
            if done is not None:
                consumer = torch.cuda.current_stream()
                consumer.wait_event(done)
                for t in frames:
                    if torch.is_tensor(t) and t.is_cuda:
                        t.record_stream(consumer)
            self.have.update(zip(range(i, i + len(frames)), frames))
            del got, frames
        return self.have[k]

    def value(self, k):
        done, values, t = self.values[k]
        if done is not None:
            done.synchronize()
        return int(values[t])

    def drop(self, k):
        del self.have[k]
        self.values.pop(k, None)

    def release(self):
        self.credits.release()

    def close(self):
        self.stop.set()
        self.credits.release()                      # wakes a reader waiting for a credit; it sees `stop` and returns
        self.thread.join()
        self.have.clear()
        self.values.clear()


def _png_head(path):
    """(h, w, bit depth) from the file's IHDR chunk, or None when it does not start like a PNG."""
    from ..png import SIGNATURE
    with open(path, 'rb') as f:
        head = f.read(25)
    if len(head) == 25 and head[:8] == SIGNATURE and head[12:16] == b'IHDR':
        w, h, depth = struct.unpack('>IIB', head[16:25])
        return int(h), int(w), int(depth)
    return None


def _imread_any(path):
    """The reference's cv.imread(name, 3) = IMREAD_COLOR | IMREAD_ANYDEPTH (uint16 for 16-bit files) as contiguous RGB."""
    import cv2 as cv
    im = cv.imread(path, cv.IMREAD_COLOR | cv.IMREAD_ANYDEPTH)
    if im is None:
        raise ValueError('inference_data_loader: cannot decode ' + path)
    return np.ascontiguousarray(im[:, :, ::-1])


def read_inputs(paths, down, device=None, threads=INFERENCE_THREADS, window_bytes=None):
    """The frames of `paths` as the reference's inference input (lib/dataloader.py:38-43), each an [h, w, 3] float32
    tensor on `device`: frame / 255, or with `down` the HR frame's GaussianBlur(sigma 1.5)[::4, ::4] / 255, bit for bit.

    Files are taken in windows of about `window_bytes` of decoded pixels (png.BATCH_BYTES).  A window's 8-bit PNGs are
    decoded by png.decode_png (on the device, or by cv2 where device_pays or the device's subset says so), its other
    files -- 16-bit PNGs, which stay uint16 as cv2 reads them, and files that are not PNGs -- by cv2 on the host and
    uploaded; then one launch per frame size and depth converts (K.frames_to_f32) or down-samples (K.gauss_blur_down4)
    the window, and its decoded frames are released.  So at most one window of input pixels is on the device at once;
    the float32 frames of the whole sequence stay there, views of one tensor per launch."""
    import torch
    from .. import png
    device = torch.device('cuda') if device is None else torch.device(device)
    window_bytes = png.BATCH_BYTES if window_bytes is None else int(window_bytes)
    heads = [_png_head(p) for p in paths]
    cost = [hd[0] * hd[1] * 3 * (2 if hd[2] > 8 else 1) if hd else os.path.getsize(p) for p, hd in zip(paths, heads)]
    convert = K.gauss_blur_down4 if down else K.frames_to_f32
    out = [None] * len(paths)
    with concurrent.futures.ThreadPoolExecutor(max_workers=max(1, int(threads))) as pool:
        for i, j in png._windows(cost, window_bytes):
            eight = [k for k in range(i, j) if heads[k] is not None and heads[k][2] <= 8]
            rest = [k for k in range(i, j) if heads[k] is None or heads[k][2] > 8]
            frames = {}
            if eight:
                frames.update(zip(eight, png.decode_png([paths[k] for k in eight], device, threads, window_bytes)))
            for k, im in zip(rest, pool.map(_imread_any, [paths[k] for k in rest])):
                frames[k] = torch.from_numpy(im).to(device)
            groups = {}
            for k in range(i, j):
                groups.setdefault((tuple(frames[k].shape), frames[k].dtype), []).append(k)
            for ks in groups.values():
                for a in range(0, len(ks), 65535):               # frames per launch
                    for k, im in zip(ks[a:a + 65535], convert([frames[k] for k in ks[a:a + 65535]])):
                        out[k] = im
            del frames
    return out


def frvsr_gpu_data_loader(HR_frames, FLAGS):
    """Device half of reference lib/dataloader.py:306-332.  HR_frames: CUDA [B,RNN_N,crop*4+8,crop*4+8,3] in [0,1]
    (the CPU queue's output).  Returns (s_inputs [B,T,crop,crop,3] in [0,1], s_targets [B,T,4crop,4crop,3] in [-1,1]):
    LR = 9x9 sigma-1.5 Gaussian stride-4 VALID; target = centre crop, preprocessed."""
    B, T, Hh, Ww, _ = HR_frames.shape
    crop = FLAGS.crop_size
    k_w_border = int(1.5 * 3.0)
    if Hh != crop * 4 + 2 * k_w_border or Ww != Hh:
        raise ValueError("frvsr_gpu_data_loader: HR frames must be %dx%d" % (crop * 4 + 2 * k_w_border, crop * 4 + 2 * k_w_border))
    flat = HR_frames.reshape(B * T, Hh, Ww, 3).contiguous()
    lr = K.gauss_down4(flat).reshape(B, T, crop, crop, 3)
    tgt = flat[:, k_w_border:k_w_border + crop * 4, k_w_border:k_w_border + crop * 4, :].contiguous()
    tgt = preprocess(tgt).reshape(B, T, crop * 4, crop * 4, 3)
    return lr, tgt


class EmptyClipSet(ValueError):
    """The scene range holds no usable clip, or fewer samples than one batch."""


# One sample's draws: scene index into HRClipLoader.clips, the RNN_N source frame numbers, int64 [RNN_N, 2] top-left
# (y, x) of each frame's window in its source frame, and the left-right flip.
ClipDraw = collections.namedtuple('ClipDraw', 'clip, frames, origin, flip')


class HRClipLoader:
    """Host half of the training input (reference lib/dataloader.py:147-273, `loadHR`; main.py flags :60-78).

    Layout: `<input_video_dir>/<input_video_pre>_%04d/col_high_%04d.png`, directories str_dir..end_dir, frames 0..max_frm;
    a directory without frame `max_frm` is skipped.  One sample = RNN_N consecutive frames starting at any of the
    max_frm - RNN_N + 1 positions; per sample, with fresh random numbers:
      * movingFirstFrame (`:206-226`): integer steps floor(U(-3.5, 4.5)) per frame, cumulated; with probability 0.3 the
        clip is replaced by crops of its FIRST frame sliding along that path (camera-motion augmentation), all of the
        size (H - y range, W - x range);
      * random_crop (`:236-249`): one tar_size x tar_size window, offsets floor(U(0, size - tar_size)), shared by the frames
        (random_crop off raises, as in the reference: clips have different resolutions);
      * flip (`:251-258`): left-right flip of every frame when a uniform draw is < 0.5.
    Batches of batch_size clips come from a per-epoch permutation (seeded by rand_seed; `shuffle_batch` in the reference is
    a thread-order-dependent shuffle buffer, which is not reproducible by design).  Under data parallelism rank r takes
    every world-th clip of the permutation.  Decoding runs on `queue_thread` worker threads, `prefetch` batches ahead;
    every sample's augmentation is a function of (rand_seed, epoch, sample index) only, so a run is reproducible whatever
    the thread timing.  Output: float32 [B, RNN_N, tar_size, tar_size, 3] in [0, 1] (pinned when CUDA is available) for
    `frvsr_gpu_data_loader`.

    `dirs` = (first, last) overrides str_dir..end_dir and `salt` != 0 moves every permutation and augmentation draw to a
    stream of its own: the validation loader (`validation_loader`, reference lib/dataloader.py:287-297) reads the held-out
    scenes end_dir+1..end_dir_val with the same augmentation, and its draws never repeat the training loader's.  With the
    defaults the training batches are those of a loader without these arguments, byte for byte.

    sample() = assemble(draw()): draw() makes every random choice of a sample from the frame size alone (PNG header),
    assemble() decodes and cuts the pixels; FrameStore cuts the same draws from frames held on the device."""

    def __init__(self, FLAGS, tar_size=None, rank=0, world=1, prefetch=4, dirs=None, salt=0, queue_thread=None):
        self.F = FLAGS
        self.tar_size = tar_size if tar_size is not None else FLAGS.crop_size * 4 + int(1.5 * 3.0) * 2
        self.rank, self.world, self.prefetch = rank, world, max(1, prefetch)
        self.salt = [int(salt)] if salt else []       # last seed word; salt 0 leaves the training seeds as they were
        self.queue_thread = int(FLAGS.queue_thread if queue_thread is None else queue_thread)
        self._sizes, self._order_cache = {}, None
        first, last = dirs if dirs is not None else (FLAGS.str_dir, FLAGS.end_dir)
        if FLAGS.input_video_dir == '':
            raise ValueError('Video input directory input_video_dir is not provided')
        if not os.path.exists(FLAGS.input_video_dir):
            raise ValueError('Video input directory not found')
        self.clips = []
        for dir_i in range(first, last + 1):
            d = os.path.join(FLAGS.input_video_dir, '%s_%04d' % (FLAGS.input_video_pre, dir_i))
            if not os.path.exists(d):
                continue
            if not os.path.exists(os.path.join(d, 'col_high_%04d.png' % FLAGS.max_frm)):
                print("Skip %s, since foler doesn't contain enough frames!" % d)
                continue
            self.clips.append(d)
        self.windows = FLAGS.max_frm - FLAGS.RNN_N + 1
        if not self.clips or self.windows <= 0:
            raise EmptyClipSet('No frame files in the video input directory')
        self.image_count = len(self.clips) * self.windows
        self.steps_per_epoch = self.image_count // (FLAGS.batch_size * world)
        if self.steps_per_epoch == 0:
            raise EmptyClipSet('HRClipLoader: %d samples cannot fill one batch of %d x %d ranks'
                             % (self.image_count, FLAGS.batch_size, world))
        print('Sequenced batches: {}, sequence length: {}'.format(self.image_count, FLAGS.RNN_N))

    def __len__(self):
        return self.image_count

    @staticmethod
    def decode(path):
        """A frame as uint8 RGB [H, W, 3] (a view of cv2's BGR array); decode_png of the reference."""
        import cv2 as cv
        im = cv.imread(path, cv.IMREAD_COLOR)
        if im is None:
            raise ValueError('HRClipLoader: cannot decode ' + path)
        return im[:, :, ::-1]

    def frame_path(self, clip, frame):
        return os.path.join(self.clips[clip], 'col_high_%04d.png' % frame)

    def frame_size(self, path):
        """(height, width) of a frame, from its PNG header (a file that is not a PNG is decoded); cached per path."""
        hw = self._sizes.get(path)
        if hw is None:
            with open(path, 'rb') as f:
                head = f.read(24)
            if len(head) == 24 and head[:8] == b'\x89PNG\r\n\x1a\n' and head[12:16] == b'IHDR':
                w, h = struct.unpack('>II', head[16:24])
                hw = (int(h), int(w))
            else:
                hw = tuple(self.decode(path).shape[:2])
            self._sizes[path] = hw
        return hw

    def draw(self, index, epoch=0):
        """The random half of sample(): which frames, where, flipped or not -- a ClipDraw; deterministic in
        (rand_seed, epoch, index).  Needs the frame size only, which comes from the PNG header."""
        F, T, tar = self.F, self.F.RNN_N, self.tar_size
        ci, start = index // self.windows, index % self.windows
        rng = np.random.default_rng([int(F.rand_seed) & 0x7FFFFFFF, int(epoch), int(index)] + self.salt)
        moving = False
        if F.movingFirstFrame:
            step = np.floor(rng.uniform(-3.5, 4.5, size=(T, 2))).astype(np.int64)
            pos = np.cumsum(step, axis=0) - step                      # exclusive cumulative sum: relative positions
            span = pos.max(axis=0) - pos.min(axis=0)                  # [shrink x, shrink y]
            lefttop = pos - pos.min(axis=0)
            moving = not (rng.uniform() < 0.7)
        if not F.random_crop:
            raise Exception('Not implemented')      # reference :250: train data have different resolutions, crop is necessary
        h, w = self.frame_size(self.frame_path(ci, start))
        if moving:      # crops of the first frame sliding along the path, each (h - shrink y) x (w - shrink x)
            h, w = h - int(span[1]), w - int(span[0])
            frames, origin = (start,) * T, lefttop[:, ::-1].astype(np.int64)
        else:
            frames, origin = tuple(range(start, start + T)), np.zeros((T, 2), np.int64)
        if h < tar or w < tar:
            raise ValueError('HRClipLoader: %s frames (%dx%d after augmentation) are smaller than the %d-pixel crop'
                             % (self.clips[ci], h, w, tar))
        off_w = int(np.floor(rng.uniform(0, float(w) - tar)))
        off_h = int(np.floor(rng.uniform(0, float(h) - tar)))
        flip = bool(getattr(F, 'flip', True) and rng.uniform() < 0.5)
        return ClipDraw(ci, frames, origin + np.array([off_h, off_w], np.int64), flip)

    def assemble(self, d):
        """The pixel half of sample(): the tar x tar windows of a ClipDraw, flipped when drawn so, as float32 u8 / 255
        (convert_image_dtype: numpy's correctly rounded float32 division)."""
        tar = self.tar_size
        img = {f: self.decode(self.frame_path(d.clip, f)) for f in sorted(set(d.frames))}
        out = np.stack([img[f][y:y + tar, x:x + tar] for f, (y, x) in zip(d.frames, d.origin.tolist())])
        if d.flip:
            out = out[:, :, ::-1]
        return np.divide(out.astype(np.float32), np.float32(255.0))

    def sample(self, index, epoch=0):
        """One augmented clip [RNN_N, tar, tar, 3]; deterministic in (rand_seed, epoch, index)."""
        return self.assemble(self.draw(index, epoch))

    def _order(self, epoch):
        cached = self._order_cache
        if cached is not None and cached[0] == epoch:
            return cached[1]
        perm = np.random.default_rng([int(self.F.rand_seed) & 0x7FFFFFFF, 0x5EED, int(epoch)] + self.salt).permutation(self.image_count)
        order = perm[self.rank::self.world]
        self._order_cache = (epoch, order)
        return order

    def _indices(self, step):
        epoch, k = divmod(step, self.steps_per_epoch)
        B = self.F.batch_size
        return epoch, self._order(epoch)[k * B:(k + 1) * B]

    def _empty_batch(self):
        import torch
        out = torch.empty((self.F.batch_size, self.F.RNN_N, self.tar_size, self.tar_size, 3), dtype=torch.float32)
        return out.pin_memory() if torch.cuda.is_available() else out

    def batch(self, step):
        """Batch number `step` of the endless stream `batches()` yields, decoded on the calling thread."""
        import torch
        epoch, idx = self._indices(step)
        out = self._empty_batch()
        for b, i in enumerate(idx):
            out[b] = torch.from_numpy(self.sample(int(i), epoch))
        return out

    def batches(self, start_step=0):
        """Endless iterator over torch tensors [B, RNN_N, tar, tar, 3]; `start_step` lets a resumed run skip ahead."""
        import torch
        build = self._indices
        with concurrent.futures.ThreadPoolExecutor(max_workers=max(1, self.queue_thread)) as pool:
            pending = collections.deque()

            def submit(step):
                epoch, idx = build(step)
                pending.append([pool.submit(self.sample, int(i), epoch) for i in idx])
            step = start_step
            for s in range(step, step + self.prefetch):
                submit(s)
            while True:
                futs = pending.popleft()
                submit(step + self.prefetch)
                out = self._empty_batch()
                for b, f in enumerate(futs):
                    out[b] = torch.from_numpy(f.result())
                yield out
                step += 1


VALIDATION_SALT = 0x7A1D


def validation_loader(FLAGS):
    """The held-out scenes end_dir+1 .. end_dir_val (reference lib/dataloader.py:287-297: same loader and augmentation,
    queue_thread = 1) as (HRClipLoader, None), or (None, reason) when that range holds no usable scene or fewer samples
    than one batch -- the reference raises there; here training goes on without validation."""
    try:
        return HRClipLoader(FLAGS, dirs=(FLAGS.end_dir + 1, FLAGS.end_dir_val), salt=VALIDATION_SALT, queue_thread=1), None
    except EmptyClipSet as e:
        return None, '%s (scenes %s_%04d .. %s_%04d)' % (e, FLAGS.input_video_pre, FLAGS.end_dir + 1,
                                                         FLAGS.input_video_pre, FLAGS.end_dir_val)


class FrameStore:
    """Every frame of the scenes of one or more HRClipLoaders (training and held-out scenes), decoded once into one flat
    uint8 RGB device buffer, and the batches of those loaders cut from it on the GPU.

    Frame i sits at byte offsets[i] with shape sizes[i] = (H, W); sizes come from the PNG headers, so the offsets are known
    before anything is decoded, and scenes may differ in size.  `queue_thread` host threads read the files and pack
    their compressed streams into a pinned stage; the device decodes them in chunks of about `chunk_bytes` straight
    into the store (tecogan_b200/png.py::decode_png_into), and a file outside its PNG subset is decoded on the host.  With world > 1 (an initialised torch.distributed group
    whose backend can broadcast `device` tensors: NCCL under torchrun) rank r decodes the r-th contiguous share of the
    frames and broadcasts it, so every rank holds the whole store after 1/world of the decoding.

    placement='host' keeps the frames in host memory instead (tecogan_b200/hostmem.py::shared_mapping): one memfd mapping
    per node, shared by the node's ranks, page-locked and mapped into the device's address space.  Each rank of a node
    decodes its contiguous share of the frames on its own device, `chunk_bytes` at a time, and copies each chunk into the
    mapping; a barrier follows.  The batches are cut over PCIe by teco_gather_clips_host_u8.  close() releases the
    mapping (unregister, then unmap).

    batch(step) is HRClipLoader.batch(step) of the first loader, uploaded to `device`, bit for bit: the same draws
    (HRClipLoader.draw: permutation, epochs, rank shard, salt) and the same pixels, cut by teco_gather_clips_u8.
    view(loader) is the same store serving another of the loaders it was built from (the validation scenes)."""

    def __init__(self, loaders, device, rank=0, world=1, queue_thread=None, chunk_bytes=256 << 20, placement='device'):
        import torch
        loaders = list(loaders)
        self.loader, self.device = loaders[0], torch.device(device)
        paths, self._bases = [], {}
        index = {}
        for L in loaders:
            base = np.empty(len(L.clips), np.int64)
            for ci in range(len(L.clips)):
                first = L.frame_path(ci, 0)
                if first not in index:               # a scene two loaders share is stored once
                    index[first] = len(paths)
                    paths += [L.frame_path(ci, f) for f in range(L.F.max_frm + 1)]
                base[ci] = index[first]
            self._bases[id(L)] = base
        hw = np.array([self.loader.frame_size(p) for p in paths], np.int64).reshape(-1, 2)
        for L in loaders[1:]:                        # the views' draws read frame sizes through their own loader
            L._sizes.update(zip(paths, map(tuple, hw.tolist())))
        nbytes = hw[:, 0] * hw[:, 1] * 3
        self.sizes, self.paths = hw, paths
        self.offsets = np.concatenate([[0], np.cumsum(nbytes)]).astype(np.int64)
        self.nbytes = int(self.offsets[-1])
        t0 = time.time()
        if placement not in ('device', 'host'):
            raise ValueError("FrameStore: placement is 'device' or 'host', got %r" % (placement,))
        self.placement = placement
        threads = max(1, int(self.loader.queue_thread if queue_thread is None else queue_thread))
        if placement == 'host':
            self._build_host(paths, rank, world, threads, chunk_bytes)
            self.build_seconds = time.time() - t0
            return
        self.buf = torch.empty(self.nbytes, dtype=torch.uint8, device=self.device)
        shares = frame_shares(len(paths), world)
        self._decode(paths, *shares[rank], threads, chunk_bytes)
        if world > 1:
            import torch.distributed as dist
            for r, (a, b) in enumerate(shares):
                if b > a:
                    dist.broadcast(self.buf[int(self.offsets[a]):int(self.offsets[b])], src=r)
        torch.cuda.synchronize(self.device)
        self.build_seconds = time.time() - t0

    @staticmethod
    def estimate_bytes(loaders):
        """Bytes a FrameStore of these loaders would take, from the PNG headers alone (nothing decoded)."""
        seen, total = set(), 0
        for L in loaders:
            for ci in range(len(L.clips)):
                if L.clips[ci] in seen:
                    continue
                seen.add(L.clips[ci])
                for f in range(L.F.max_frm + 1):
                    h, w = L.frame_size(L.frame_path(ci, f))
                    total += h * w * 3
        return total

    def _build_host(self, paths, rank, world, threads, chunk_bytes):
        """The host placement: the node's shared mapping, this rank's share of it decoded on the device chunk by chunk
        and copied in, then a barrier."""
        import torch
        from ..hostmem import shared_mapping
        with torch.cuda.device(self.device):         # registered on, and synchronised on close with, this device
            self._host, node = shared_mapping(self.nbytes, rank, world)
        try:
            self.buf = torch.from_numpy(self._host.array())
            a, b = frame_shares(len(paths), len(node))[node.index(rank)]
            while a < b:
                end = a + 1
                while end < b and self.offsets[end + 1] - self.offsets[a] <= chunk_bytes:
                    end += 1
                lo, hi = int(self.offsets[a]), int(self.offsets[end])
                stage = torch.empty(hi - lo, dtype=torch.uint8, device=self.device)
                self._decode(paths, a, end, threads, chunk_bytes, stage, self.offsets[a:end] - lo)
                self.buf[lo:hi].copy_(stage)
                a = end
            torch.cuda.synchronize(self.device)
            if world > 1:
                import torch.distributed as dist
                dist.barrier()
        except BaseException:
            self.close()
            raise

    def close(self):
        """Releases a host placement's mapping: waits for the store's device, unregisters the mapping, then unmaps it
        (errors are raised).  The store and its views must not be used afterwards.  A device placement's memory is freed
        with the store."""
        host = self.__dict__.pop('_host', None)
        if host is not None:
            self.buf = None
            host.close()

    def _decode(self, paths, a, b, threads, chunk_bytes, buf=None, offsets=None):
        """Frames a..b-1 into self.buf (or into `buf` at `offsets`): host threads read the files and pack their
        compressed streams, the device decodes them in chunks of about chunk_bytes (tecogan_b200.png.decode_png_into);
        a file the device does not take is decoded on the host by the loader and copied into its slot."""
        from ..png import decode_png_into
        if b <= a:
            return
        expect = {paths[k]: tuple(int(v) for v in self.sizes[k]) for k in range(a, b)}

        def host(path):
            im = self.loader.decode(path)
            h, w = expect[path]
            if im.shape[:2] != (h, w):
                raise ValueError('FrameStore: %s decodes to %dx%d, its header says %dx%d' % (path, im.shape[0], im.shape[1], h, w))
            return im
        decode_png_into(paths[a:b], self.buf if buf is None else buf, self.offsets[a:b] if offsets is None else offsets,
                        self.sizes[a:b], threads=threads, batch_bytes=chunk_bytes, host_decode=host)

    def view(self, loader):
        """This store serving `loader`, one of the loaders it was built from."""
        if id(loader) not in self._bases:
            raise ValueError('FrameStore.view: the store was not built from this loader')
        v = object.__new__(FrameStore)
        v.__dict__.update(self.__dict__)
        v.loader = loader
        return v

    def table(self, step):
        """int64 [B * RNN_N, 3] rows of teco_gather_clips_u8 for batch `step` of this store's loader."""
        L = self.loader
        tar = L.tar_size
        epoch, idx = L._indices(step)
        base = self._bases[id(L)]
        fid, org, flip = [], [], []
        for i in idx:
            d = L.draw(int(i), epoch)
            fid.append(base[d.clip] + np.asarray(d.frames, np.int64))
            org.append(d.origin)
            flip.append(np.full(len(d.frames), d.flip, np.int64))
        fid, org, flip = np.concatenate(fid), np.concatenate(org), np.concatenate(flip)
        h, w = self.sizes[fid, 0], self.sizes[fid, 1]
        if (org < 0).any() or (org[:, 0] + tar > h).any() or (org[:, 1] + tar > w).any():
            bad = int(np.flatnonzero((org[:, 0] + tar > h) | (org[:, 1] + tar > w) | (org < 0).any(axis=1))[0])
            raise ValueError('FrameStore: a %d-pixel window at %s does not fit in %s (%dx%d)'
                             % (tar, org[bad].tolist(), self.paths[fid[bad]], h[bad], w[bad]))
        return np.stack([self.offsets[fid] + (org[:, 0] * w + org[:, 1]) * 3, w * 3, flip], axis=1)

    def _gather(self, tbl):
        import torch
        L = self.loader
        t = torch.from_numpy(tbl).pin_memory().to(self.device, non_blocking=True)
        if self.placement == 'host':
            out = K.gather_clips_host_u8(self._host.dev_addr, t, L.tar_size)
        else:
            out = K.gather_clips_u8(self.buf, t, L.tar_size)
        return out.reshape(L.F.batch_size, L.F.RNN_N, L.tar_size, L.tar_size, 3)

    def batch(self, step):
        """Batch number `step` of the loader, fp32 [B, RNN_N, tar, tar, 3] on the device: HRClipLoader.batch(step)."""
        return self._gather(self.table(step))

    def batches(self, start_step=0, prefetch=4):
        """Endless iterator over batch(start_step), batch(start_step + 1), ...; the draws of the next `prefetch` steps are
        made on a worker thread while the device works.  In host placement the gather of step k + 1 is enqueued on a
        stream of its own as soon as batch k is handed out, so its PCIe reads overlap the caller's work on batch k; the
        caller's stream waits for each batch, and record_stream keeps its memory from being reused while it is held."""
        import torch
        with concurrent.futures.ThreadPoolExecutor(max_workers=1) as pool:
            pending = collections.deque(pool.submit(self.table, s) for s in range(start_step, start_step + prefetch))
            step = start_step
            if self.placement != 'host':
                while True:
                    tbl = pending.popleft().result()
                    pending.append(pool.submit(self.table, step + prefetch))
                    yield self._gather(tbl)
                    step += 1
            side, drawn = torch.cuda.Stream(self.device), itertools.count(start_step + prefetch)

            def launch():
                tbl = pending.popleft().result()
                pending.append(pool.submit(self.table, next(drawn)))
                with torch.cuda.stream(side):
                    out = self._gather(tbl)
                    done = torch.cuda.Event()
                    done.record(side)
                return out, done
            ahead = launch()
            while True:
                out, done = ahead
                consumer = torch.cuda.current_stream(self.device)
                consumer.wait_event(done)
                out.record_stream(consumer)
                ahead = launch()
                yield out
                step += 1

    def checksum(self):
        """SHA-256 of the store's bytes (to compare the stores of several ranks)."""
        import hashlib
        return hashlib.sha256(self.buf.cpu().numpy().tobytes()).hexdigest()


def frame_shares(n, world):
    """Contiguous [a, b) frame ranges, one per rank, covering 0..n with sizes differing by at most one."""
    cuts = [n * r // world for r in range(world + 1)]
    return [(cuts[r], cuts[r + 1]) for r in range(world)]
