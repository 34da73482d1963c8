"""The training data of the reference's dataPrepare.py, made from local videos on the GPU: each listed scene becomes a
folder `scene_%04d/` of `col_high_%04d.png` frames, every frame decoded by cv2, down-sampled by
cv2.resize(fx=0.5, fy=0.5, INTER_AREA) and written by cv2.imwrite in the reference -- here down-sampled by
teco_area_half_u8 and PNG-encoded by teco_png_encode_rgb8, byte for byte the same files (DESIGN.md section 4.10).

The control flow, the scene numbering and the printed lines are the reference's (dataPrepare.py:103-152).  There is no
download: the source of video <id> is the one file `<disk_path>/<id>.<ext>` that youtube-dl would have left there, and a
missing one is skipped as the reference skips a failed download.

One intended deviation in how frames are decoded: the reference seeks before every frame (lib/data/video.py:168-170);
here each scene seeks once, to its start frame, and reads its frames in sequence.  On a container whose seeking is exact
the frames are the same; where seeking is inexact, the reference's frames are not well defined either.

`dataPrepare.py --scene_threshold T` (DESIGN.md section 4.14) makes the table instead of taking the reference's: scan()
decodes every video in disk_path, finds its hard cuts on the GPU with `main.py --scene_threshold`'s rule and cuts
--duration-frame scenes that hold no cut; prepare() then writes them as it writes the table's, reading those videos in
sequence instead of seeking.
"""
import itertools
import json
import os
import threading

LINK_PATH = "https://vimeo.com/"        # printed as the reference prints it; nothing is fetched
MIN_SIDE = 400                          # videos under 400 px on either side are skipped (reference dataPrepare.py:135)
WINDOW_BYTES = 64 << 20                 # decoded source frames per staging buffer (at least one frame)
STAGING = 2                             # pinned staging buffers per worker: one filling, one being uploaded
# The files --scene_threshold takes as videos, by lower-cased extension.
VIDEO_EXTS = (".mp4", ".m4v", ".mov", ".mkv", ".webm", ".avi", ".mpg", ".mpeg", ".ts")

# The reference's vimeo id -> start frames table (dataPrepare.py:26-62), in its order: scene numbers follow it.  The
# frames are chosen so that no scene switch falls inside 120 frames.
VIDEOS = {
    "121649159": [0, 310, 460, 720, 860],
    "40439273": [90, 520, 700, 1760, 2920, 3120, 3450, 4750, 4950, 5220, 6500, 6900, 9420, 9750],
    "87389090": [100, 300, 500, 800, 1000, 1200, 1500, 1900, 2050, 2450, 2900],
    "335874600": [287, 308, 621, 1308, 1538, 1768, 2036, 2181, 2544, 2749, 2867, 3404, 3543, 3842, 4318, 4439, 4711, 4900,
                  7784, 8811, 9450],
    "114053015": [30, 1150, 2160, 2340, 3190, 3555],
    "160578133": [550, 940, 1229, 1460, 2220, 2900, 3180, 4080, 4340, 4612, 4935, 5142, 5350, 5533, 7068],
    "148058982": [80, 730, 970, 1230, 1470, 1740],
    "150225201": [0, 560, 1220, 1590, 1780],
    "145096806": [0, 300, 550, 800, 980, 1500],
    "125621327": [240, 900, 1040, 1300, 1970, 2130, 2530, 3020, 3300, 3620, 3830, 4300, 4700, 4960],
    "162166758": [120, 350, 540, 750, 950, 1130, 1320, 1530, 1730, 1930],
    "115829238": [140, 450, 670, 910, 1100, 1380, 1520, 1720],
    "159455925": [40, 340, 490, 650, 850, 1180, 1500, 1800, 2000, 2300, 2500, 2800, 3200],
    "193873193": [0, 280, 1720],
    "133842385": [300, 430, 970, 1470, 1740, 2110, 2240, 2760, 3080, 3210, 3400, 3600],
    "97692560": [0, 210, 620, 930, 1100, 1460, 1710, 2400, 2690, 3200, 3400, 3560, 3780],
    "142480565": [835, 1380, 1520, 1700, 2370, 4880],
    "174952003": [480, 680, 925, 1050, 1200, 1380, 1600, 1800, 2100, 2350, 2480, 2680, 3000, 3200, 3460, 4500, 4780, 5040,
                  5630, 5830, 6400, 6680, 7300, 7500, 7800],
    "165643973": [300, 600, 1000, 1500, 1700, 1900, 2280, 2600, 2950, 3200, 3500, 3900, 4300, 4500],
    "163736142": [120, 400, 700, 1000, 1300, 1500, 1750, 2150, 2390, 2550, 3100, 3400, 3800, 4100, 4400, 4800, 5100, 5500,
                  5800, 6300],
    "189872577": [0, 170, 340, 4380, 4640, 5140, 7300, 7470, 7620, 7860, 9190, 9370],
    "181180995": [30, 160, 400, 660, 990, 2560, 2780, 3320, 3610, 5860, 6450, 7260, 7440, 8830, 9020, 9220, 9390],
    "167892347": [220, 1540, 2120, 2430, 5570, 6380, 6740],
    "146484162": [1770, 2240, 3000, 4800, 4980, 5420, 6800],
    "204313990": [110],
    "169958461": [140, 700, 1000, 1430, 1630, 1900, 2400, 2600, 2800, 3000, 3200, 3600, 3900, 4200, 4600, 5000, 5700, 6000,
                  6400, 6800, 7100, 7600, 7900, 8200],
    "198634890": [200, 320, 440, 1200, 1320, 1560, 1680, 1800, 1920, 3445],
    "89936769": [1260, 1380, 1880],
}


def source_file(disk_path, vid):
    """The source of video `vid`: the one regular file in disk_path whose name without its extension is `vid`, or None
    when there is none or more than one (the reference's youtube-dl names it <id>.<ext>)."""
    try:
        names = os.listdir(disk_path)
    except OSError:
        return None
    hits = [n for n in names if os.path.splitext(n)[0] == vid and os.path.isfile(os.path.join(disk_path, n))]
    return os.path.join(disk_path, hits[0]) if len(hits) == 1 else None


def list_sources(disk_path):
    """The videos of --scene_threshold: the regular files directly in disk_path (no recursion) whose lower-cased
    extension is in VIDEO_EXTS, in sorted file-name order -> [(stem, [paths])], one entry per stem at its first file.
    A stem with more than one path is ambiguous, as source_file finds it, and is skipped by scan()."""
    groups = {}
    for name in sorted(os.listdir(disk_path)):
        path = os.path.join(disk_path, name)
        stem, ext = os.path.splitext(name)
        if ext.lower() in VIDEO_EXTS and os.path.isfile(path):
            groups.setdefault(stem, []).append(path)
    return list(groups.items())


def video_size(path):
    """(width, height) by CAP_PROP_FRAME_WIDTH / HEIGHT, or None when cv2 cannot open the file."""
    import cv2
    cam = cv2.VideoCapture(path)
    try:
        if not cam.isOpened():
            return None
        return int(cam.get(cv2.CAP_PROP_FRAME_WIDTH)), int(cam.get(cv2.CAP_PROP_FRAME_HEIGHT))
    finally:
        cam.release()


def scene_frames(path, starts, duration, seek=True):
    """The frames of `path` the scenes need, in order: for each start frame, one seek and `duration` sequential reads
    -> (scene index, frame index, BGR uint8 frame).  A frame that cannot be read raises RuntimeError (the reference's
    cv.resize fails on it).  Without `seek` the video is read in sequence from frame 0, the frames before each scene
    passed over with grab(): then the scenes must be in order and disjoint (else ValueError)."""
    import cv2
    cam = cv2.VideoCapture(path)
    try:
        if not cam.isOpened():
            raise RuntimeError("cannot open %s" % path)
        pos = 0                                  # the next frame read, without seek
        for k, start in enumerate(starts):
            if seek:
                cam.set(cv2.CAP_PROP_POS_FRAMES, start)
            elif start < pos:
                raise ValueError("%s: scene at frame %d overlaps the one before (read to frame %d)" % (path, start, pos))
            else:
                for skipped in range(pos, start):
                    if not cam.grab():
                        raise RuntimeError("%s: cannot read frame %d" % (path, skipped))
            pos = start + duration
            for i in range(duration):
                ok, frame = cam.read()
                if not ok:
                    raise RuntimeError("%s: cannot read frame %d" % (path, start + i))
                yield k, i, frame
    finally:
        cam.release()


class _Staging:
    """Decoded frames of one video on their way to the device: STAGING pinned buffers of `n` frames each, filled in
    turn on the host; a full one is uploaded on the worker's stream, down-sampled in one teco_area_half_u8 launch into
    RGB and handed on as a window: handoff(frames, tags), frames the window's uint8 [m, h', w', 3] device frames, free
    again once the work handoff enqueues on the stream has read them, and tags what add() was given with each.  A pinned
    buffer is filled again only once its upload is done."""

    def __init__(self, h, w, n, device, handoff):
        import torch
        from . import kernels as K
        self.h, self.w, self.n, self.handoff = h, w, n, handoff
        self.host = [torch.empty((n, h, w, 3), dtype=torch.uint8, pin_memory=True) for _ in range(STAGING)]
        self.uploaded = [None] * STAGING
        self.dev = torch.empty((n, h, w, 3), dtype=torch.uint8, device=device)
        self.out = torch.empty((n, K.area_half_size(h), K.area_half_size(w), 3), dtype=torch.uint8, device=device)
        self.cur, self.tags = 0, []

    def add(self, frame, tag):
        if frame.shape != (self.h, self.w, 3) or frame.dtype.name != "uint8":
            raise ValueError("%s: frame of %s %s in a video of %dx%d uint8 frames"
                             % (tag, frame.dtype, frame.shape, self.w, self.h))
        if not self.tags and self.uploaded[self.cur] is not None:
            self.uploaded[self.cur].synchronize()
        self.host[self.cur][len(self.tags)].numpy()[...] = frame
        self.tags.append(tag)
        if len(self.tags) == self.n:
            self.flush()

    def flush(self):
        import torch
        from . import kernels as K
        m = len(self.tags)
        if not m:
            return
        self.dev[:m].copy_(self.host[self.cur][:m], non_blocking=True)
        ev = torch.cuda.Event()
        ev.record()
        self.uploaded[self.cur] = ev
        K.area_half(self.dev[:m], swap_rb=True, out=self.out[:m])
        self.handoff(self.out[:m], self.tags)
        self.tags = []
        self.cur = (self.cur + 1) % STAGING


def prepare_video(path, scenes, duration, device, stop=None, seek=True):
    """Write the scenes of one video: scenes is [(scene directory, start frame)], each directory existing.  Runs on a
    worker thread with a CUDA stream of its own; returns early once `stop` is set.  Every thread it starts is joined
    before it returns or raises.  Without `seek` the video is read in sequence (scene_frames)."""
    import torch
    from .lib.writer import FrameWriter
    from . import kernels as K
    torch.cuda.set_device(device)
    stream = torch.cuda.Stream(device=device)
    writer = stage = None
    frames = scene_frames(path, [s for _, s in scenes], duration, seek=seek)

    def write(window, paths):
        for f, p in zip(window, paths):
            writer.put(f, p)                     # copied to a writer slot on this stream: f is free after the put
    try:
        with torch.cuda.stream(stream):
            for k, i, frame in frames:
                if stop is not None and stop.is_set():
                    return
                if stage is None:
                    h, w = frame.shape[:2]
                    writer = FrameWriter(K.area_half_size(h), K.area_half_size(w), device)
                    n = max(1, min(duration * len(scenes), WINDOW_BYTES // (3 * h * w)))
                    stage = _Staging(h, w, n, device, write)
                stage.add(frame, os.path.join(scenes[k][0], "col_high_%04d.png" % i))
            if stage is not None:
                stage.flush()
    finally:
        frames.close()
        if writer is not None:
            writer.close()
        stream.synchronize()
    if writer is not None and writer.error is not None:
        raise writer.error


def cuda_device(device=None):
    """The torch.device the frames are made on: `device`, by default the current CUDA device.  There is no host path."""
    import torch
    if not torch.cuda.is_available():
        raise RuntimeError("dataPrepare needs a CUDA device: frames are down-sampled and encoded on the GPU")
    dev = torch.device("cuda" if device is None else device)
    return dev if dev.index is not None else torch.device("cuda", torch.cuda.current_device())


def _in_order(work, jobs, threads, done):
    """work(*job, stop) for every job on up to `threads` worker threads ("dataPrepare"), and done(k, result) on this
    thread for k = 0, 1, ... in job order, each as soon as that job and every one before it have finished.  An error on
    any worker stops the others (`stop` is set, jobs not started are cancelled) and is raised here once every worker is
    joined."""
    import concurrent.futures as cf
    stop = threading.Event()
    pool = cf.ThreadPoolExecutor(max_workers=max(1, threads), thread_name_prefix="dataPrepare")
    futures = []
    try:
        futures = [pool.submit(work, *job, stop) for job in jobs]
        pending, k = set(futures), 0
        while k < len(futures):
            finished, pending = cf.wait(pending, return_when=cf.FIRST_EXCEPTION)
            for f in finished:
                f.result()                       # raises a worker's error
            while k < len(futures) and futures[k].done():
                done(k, futures[k].result())
                k += 1
    except BaseException:
        stop.set()
        for f in futures:
            f.cancel()
        raise
    finally:
        pool.shutdown(wait=True)


def prepare(videos, disk_path, start_id, duration, save_frames=True, remove=False, threads=4, device=None,
            sources=None):
    """The reference's main loop (dataPrepare.py:103-152) over `videos`, an {id: [start frames]} table in scene order.

    A video is valid when its source file (source_file) opens in cv2 and is at least MIN_SIDE on both sides; scene
    numbers start at start_id and advance once per start frame of every valid video.  With save_frames, the scenes of up
    to `threads` videos are made at once (prepare_video, on `device`, default the current CUDA device) and, with
    `remove`, each source is deleted once its scenes are written; without it nothing is written and the lines say what
    would be done.  An error on any worker stops the others and is raised here once every worker is joined.

    `sources` ({id: path}, from scan) gives every video's file instead: its path is printed in place of the link, and
    it is read in sequence, without seeking (its start frames are in order and its scenes disjoint).
    -> the number of valid videos."""
    cur_id, valid_video = start_id, 0
    print("Try loading %dx%d." % (sum(len(v) for v in videos.values()), duration))
    jobs = []
    for vid, starts in videos.items():
        link = LINK_PATH + vid if sources is None else sources[vid]
        print(link)
        path = source_file(disk_path, vid) if sources is None else sources[vid]
        size = video_size(path) if path is not None else None
        if size is None:
            print("Skipped invalid link or other error:" + link)
            continue
        width, height = size
        if width < MIN_SIDE or height < MIN_SIDE:
            print("Skipped videos of small size %dx%d" % (width, height))
            continue
        valid_video += 1
        scenes = []
        for start_fr in starts:
            tar_dir = os.path.join(disk_path, "scene_%04d/" % cur_id)
            if save_frames:
                os.makedirs(tar_dir, exist_ok=True)
            print("folder %s: %dx[%d,%d]//2 at frame %d of %s" % (tar_dir, duration, width, height, start_fr, path))
            scenes.append((tar_dir, start_fr))
            cur_id += 1
        jobs.append((path, scenes))

    if save_frames and jobs:
        dev = cuda_device(device)
        in_sequence = {} if sources is None else {"seek": False}

        def work(path, scenes, stop):
            prepare_video(path, scenes, duration, dev, stop, **in_sequence)

        def written(k, _):
            if remove:
                print("remove ", jobs[k][0])
                os.remove(jobs[k][0])
        _in_order(work, jobs, threads, written)

    print("Done: get %d valid folders with %d frames from %d videos." % (cur_id - start_id, duration, valid_video))
    return valid_video


# ---- `dataPrepare.py --scene_threshold T`: the table made from the videos themselves (DESIGN.md section 4.14) ---------

def scene_starts(scores, threshold, duration):
    """The scenes of a video of len(scores) frames.  Frame i >= 1 starts a shot iff scores[i] >= threshold; frame 0
    always starts one (scores[0] is not read).  A shot of frames [c, e) gives the disjoint windows [c + k duration,
    c + (k + 1) duration) that fit inside it, and the rest of the shot is dropped.  -> the windows' start frames,
    ascending."""
    if duration < 1:
        raise ValueError("scene duration must be >= 1, got %d" % duration)
    bounds = [0] + [i for i in range(1, len(scores)) if scores[i] >= threshold] + [len(scores)]
    return [s for c, e in zip(bounds, bounds[1:]) for s in range(c, e - duration + 1, duration)]


def frame_scores(sads, values):
    """Each frame's cut score from the SAD of its halved frame to the one before (sads[0] = 0: frame 0 has none), by
    `main.py --scene_threshold`'s rule (lib/dataloader.py::scene_score, mafd_0 = 0) over `values` = 3 h' w' bytes."""
    from .lib.dataloader import scene_score
    scores, mafd = [], 0.0
    for sad in sads:
        mafd, score = scene_score(sad, values, mafd)
        scores.append(score)
    return scores


def format_table(table):
    """An {id: [start frames]} table in the reference's syntax (its dataPrepare.py:26-62), so that a scan can be reviewed
    and reproduced."""
    rows = ["    %s : [%s]," % (json.dumps(k, ensure_ascii=False), ", ".join(str(s) for s in v)) for k, v in table.items()]
    return "\n".join(["video_data_dict = {"] + rows + ["}"])


class _FrameSads:
    """The scan's hand-off from _Staging: one frame_sads_u8 launch per window of halved frames, chained to the window
    before by a device copy of its last frame.  The window's n sums come back into one of STAGING pinned buffers, read
    on the host once that buffer is needed again or at the end (result), so the worker never waits on its own stream
    for the window it has just launched."""

    def __init__(self, n, shape, device):
        import torch
        self.prev = torch.empty(shape, dtype=torch.uint8, device=device)
        self.chained = False
        self.dev = torch.empty(n, dtype=torch.int64, device=device)
        self.host = [torch.empty(n, dtype=torch.int64, pin_memory=True) for _ in range(STAGING)]
        self.pending = [None] * STAGING            # (event after the copy, frames) per pinned buffer
        self.cur, self.sads = 0, []

    def __call__(self, frames, tags):
        import torch
        from . import kernels as K
        m = frames.shape[0]
        self._read(self.cur)
        K.frame_sads_u8(frames, self.prev if self.chained else None, self.dev[:m])
        self.prev.copy_(frames[m - 1])
        self.chained = True
        self.host[self.cur][:m].copy_(self.dev[:m], non_blocking=True)
        ev = torch.cuda.Event()
        ev.record()
        self.pending[self.cur] = (ev, m)
        self.cur = (self.cur + 1) % STAGING

    def _read(self, j):
        if self.pending[j] is not None:
            ev, m = self.pending[j]
            ev.synchronize()
            self.sads.extend(self.host[j][:m].tolist())
            self.pending[j] = None

    def result(self):
        for k in range(STAGING):                   # oldest first
            self._read((self.cur + k) % STAGING)
        return self.sads


def scan_video(path, device, stop=None):
    """Pass 1 of --scene_threshold on one video: every frame decoded in order from frame 0 by cv2.VideoCapture.read
    until a read fails (never a seek), halved on the device as prepare_video halves it (so the frames scored are the
    PNGs that would be written), and the SAD of each to the one before by frame_sads_u8.  Runs on a worker thread with
    a CUDA stream of its own; returns None once `stop` is set.  -> (sads, values): sads[i] the SAD of halved frames
    i - 1 and i (sads[0] = 0), one per frame decoded, and values = 3 h' w' (0 for a video without a frame)."""
    import cv2
    import torch
    from . import kernels as K
    torch.cuda.set_device(device)
    stream = torch.cuda.Stream(device=device)
    cam = cv2.VideoCapture(path)
    stage = sads = None
    try:
        if not cam.isOpened():
            raise RuntimeError("cannot open %s" % path)
        with torch.cuda.stream(stream):
            for i in itertools.count():
                if stop is not None and stop.is_set():
                    return None
                ok, frame = cam.read()
                if not ok:
                    break
                if stage is None:
                    h, w = frame.shape[:2]
                    half = (K.area_half_size(h), K.area_half_size(w), 3)
                    n = max(1, WINDOW_BYTES // (3 * h * w))
                    sads = _FrameSads(n, half, device)
                    stage = _Staging(h, w, n, device, sads)
                stage.add(frame, "%s frame %d" % (path, i))
            if stage is None:
                return [], 0
            stage.flush()
            return sads.result(), half[0] * half[1] * 3
    finally:
        cam.release()
        stream.synchronize()


def scan(disk_path, threshold, duration, threads=4, device=None):
    """Pass 1 of `dataPrepare.py --scene_threshold T`: the table of the videos in disk_path (list_sources) ->
    ({stem: [start frames]}, {stem: path}) in source order, for prepare(table, ..., sources=paths).

    A stem shared by several files, a file cv2 cannot open and a video under MIN_SIDE on either side are skipped with a
    line each.  Every other video is decoded whole and scored on up to `threads` worker threads (scan_video, on
    `device`, default the current CUDA device), and cut into scenes by scene_starts.  In source order, each video's
    path and frame count, its cuts as `main.py` prints them, and its number of scenes are printed, then the whole table
    (format_table).  A video without a scene is left out of the table.  An error on any worker stops the others and is
    raised here once every worker is joined."""
    if duration < 1:
        raise ValueError("scene duration must be >= 1, got %d" % duration)
    order, jobs = [], []                         # per source: the lines of a skipped one, or the index of its job
    for stem, paths in list_sources(disk_path):
        if len(paths) > 1:
            order.append(["Skipped %s: %d files share the name %s" % (", ".join(paths), len(paths), stem)])
            continue
        size = video_size(paths[0])
        if size is None:
            order.append([paths[0], "Skipped invalid link or other error:" + paths[0]])
        elif size[0] < MIN_SIDE or size[1] < MIN_SIDE:
            order.append([paths[0], "Skipped videos of small size %dx%d" % size])
        else:
            order.append(len(jobs))
            jobs.append((stem, paths[0]))

    table, sources, lines, shown = {}, {}, {}, [0]

    def show():                                  # print the sources in order as far as their lines are known
        while shown[0] < len(order):
            e = order[shown[0]]
            if isinstance(e, int) and e not in lines:
                return
            print("\n".join(lines.pop(e) if isinstance(e, int) else e))
            shown[0] += 1

    def scanned(k, result):
        stem, path = jobs[k]
        sads, values = result
        scores = frame_scores(sads, values)
        starts = scene_starts(scores, threshold, duration)
        lines[k] = (["%s: %d frames" % (path, len(sads))]
                    + ["scene cut before frame %d, score %.4f" % (i, s) for i, s in enumerate(scores)
                       if i > 0 and s >= threshold]
                    + ["%d scenes of %d frames" % (len(starts), duration)])
        if starts:
            table[stem], sources[stem] = starts, path
        show()

    show()
    if jobs:
        dev = cuda_device(device)
        _in_order(lambda stem, path, stop: scan_video(path, dev, stop), jobs, threads, scanned)
    show()
    print(format_table(table))
    return table, sources
