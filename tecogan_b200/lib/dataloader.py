"""Mirror of the reference's lib/dataloader.py: the inference PNG loader (lib/dataloader.py:11-50), the device half of
frvsr_gpu_data_loader (lib/dataloader.py:306-332) and -- as the caller side of the training path -- a host loader for
HR training clips (`HRClipLoader`) that follows `loadHR` + `tf.train.shuffle_batch` (lib/dataloader.py:147-273): same
directory layout, frame windows, moving-first-frame / random-crop / flip augmentation, a thread pool instead of TF queue
runners.  The validation split (lib/dataloader.py:287-296) is a second `HRClipLoader` over the held-out scenes
(`validation_loader`); it feeds the val_* summaries of main.py --mode train --summary_dir."""
import collections
import concurrent.futures
import os

import numpy as np

from .. import kernels as K
from .ops import preprocess


def inference_data_loader(FLAGS):
    """reference lib/dataloader.py:11-50: sorted PNG list -> RGB float32 /255 frames, with the hard-coded symmetric
    warm-up padding (list indices 5,4,3,2,1 prepended)."""
    filedir = FLAGS.input_dir_LR
    downSP = False
    if (FLAGS.input_dir_LR is None) or (not os.path.exists(FLAGS.input_dir_LR)):
        if (FLAGS.input_dir_HR is None) or (not os.path.exists(FLAGS.input_dir_HR)):
            raise ValueError('Input directory not found')
        filedir = FLAGS.input_dir_HR
        downSP = True
    import cv2 as cv
    names = [_ for _ in os.listdir(filedir) if _.endswith(".png")]
    names = sorted(names)
    names.sort(key=lambda f: int(''.join(list(filter(str.isdigit, f))) or -1))
    if FLAGS.input_dir_len > 0:
        names = names[:FLAGS.input_dir_len]
    image_list_LR = [os.path.join(filedir, _) for _ in names]

    def preprocess_test(name):
        im = cv.imread(name, 3).astype(np.float32)[:, :, ::-1]
        if downSP:
            icol_blur = cv.GaussianBlur(im, (0, 0), sigmaX=1.5)
            im = icol_blur[::4, ::4, ::]
        return np.ascontiguousarray(im / 255.0)

    image_LR = [preprocess_test(_) for _ in image_list_LR]
    image_list_LR = image_list_LR[5:0:-1] + image_list_LR
    image_LR = image_LR[5:0:-1] + image_LR
    Data = collections.namedtuple('Data', 'paths_LR, inputs')
    return Data(paths_LR=image_list_LR, inputs=image_LR)


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
    defaults the training batches are those of a loader without these arguments, byte for byte."""

    def __init__(self, FLAGS, tar_size=None, rank=0, world=1, prefetch=4, dirs=None, salt=0, queue_thread=None):
        self.F = FLAGS
        self.tar_size = tar_size if tar_size is not None else FLAGS.crop_size * 4 + int(1.5 * 3.0) * 2
        self.rank, self.world, self.prefetch = rank, world, max(1, prefetch)
        self.salt = [int(salt)] if salt else []       # last seed word; salt 0 leaves the training seeds as they were
        self.queue_thread = int(FLAGS.queue_thread if queue_thread is None else queue_thread)
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
    def _read(path):
        import cv2 as cv
        im = cv.imread(path, cv.IMREAD_COLOR)
        if im is None:
            raise ValueError('HRClipLoader: cannot decode ' + path)
        return np.ascontiguousarray(im[:, :, ::-1]).astype(np.float32) / 255.0       # decode_png + convert_image_dtype

    def sample(self, index, epoch=0):
        """One augmented clip [RNN_N, tar, tar, 3]; deterministic in (rand_seed, epoch, index)."""
        F, T, tar = self.F, self.F.RNN_N, self.tar_size
        clip, start = self.clips[index // self.windows], index % self.windows
        rng = np.random.default_rng([int(F.rand_seed) & 0x7FFFFFFF, int(epoch), int(index)] + self.salt)
        moving = False
        if F.movingFirstFrame:
            step = np.floor(rng.uniform(-3.5, 4.5, size=(T, 2))).astype(np.int64)
            pos = np.cumsum(step, axis=0) - step                      # exclusive cumulative sum: relative positions
            span = pos.max(axis=0) - pos.min(axis=0)                  # [shrink x, shrink y]
            lefttop = pos - pos.min(axis=0)
            moving = not (rng.uniform() < 0.7)
        if moving:
            first = self._read(os.path.join(clip, 'col_high_%04d.png' % start))
            h, w = first.shape[0] - int(span[1]), first.shape[1] - int(span[0])
            frames = [first[int(lefttop[t][1]):int(lefttop[t][1]) + h, int(lefttop[t][0]):int(lefttop[t][0]) + w] for t in range(T)]
        else:
            frames = [self._read(os.path.join(clip, 'col_high_%04d.png' % (start + t))) for t in range(T)]
        if not F.random_crop:
            raise Exception('Not implemented')      # reference :250: train data have different resolutions, crop is necessary
        h, w = frames[0].shape[:2]
        if h < tar or w < tar:
            raise ValueError('HRClipLoader: %s frames (%dx%d after augmentation) are smaller than the %d-pixel crop' % (clip, h, w, tar))
        off_w = int(np.floor(rng.uniform(0, float(w) - tar)))
        off_h = int(np.floor(rng.uniform(0, float(h) - tar)))
        out = np.stack([f[off_h:off_h + tar, off_w:off_w + tar] for f in frames])
        if getattr(F, 'flip', True) and rng.uniform() < 0.5:
            out = out[:, :, ::-1]
        return np.ascontiguousarray(out, dtype=np.float32)

    def _order(self, epoch):
        perm = np.random.default_rng([int(self.F.rand_seed) & 0x7FFFFFFF, 0x5EED, int(epoch)] + self.salt).permutation(self.image_count)
        return perm[self.rank::self.world]

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
