#!/usr/bin/env python
"""Entry point mirroring the reference's main.py: same flag names (main.py:30-105), `--mode inference` follows the
per-frame loop of main.py:253-268, `--mode train` follows main.py:273-430 (TecoGAN when --ratio > 0, else FRVSR).

Differences forced by the environment, stated once:
  * weights: --checkpoint / --vgg_ckpt take TensorFlow checkpoints (V2 bundle prefix or V1 file), read WITHOUT TensorFlow by
    tecogan_b200/tf_bundle.py (format restated from its public description; no real checkpoint was available to pin it),
    a .pt file written by this program (name -> tensor, TF variable names), or `random:<seed>` for a seeded xavier
    initialisation; training saves both a .pt file and a TF V2 bundle;
  * training data: --input_video_dir is read by a thread-pool loader with the reference's directory layout and
    augmentations (tecogan_b200/lib/dataloader.py::HRClipLoader, after lib/dataloader.py:147-273) instead of TF queue
    runners; an empty flag raises as in the reference unless --synthetic_data is given (seeded synthetic HR clips and,
    without --vgg_ckpt, a seeded random frozen VGG -- for benchmarks and tests only); the device half (Gaussian
    down-sampling, crops) is the same either way.  When every frame of the training (and held-out) scenes fits in device
    memory beside training, the frames are decoded once into a device-resident frame store and the clips are cut on the
    GPU from the same draws (FrameStore; select_training_input decides after the first step), so the batches are the host
    loader's, bit for bit; when they fit in host memory instead, the store is one page-locked host copy per node, mapped
    into the device's address space and cut over PCIe;
  * --precision {bf16,fp32} selects wgmma tensor-core or fp32 CUDA-core convolutions for inference;
    --train_precision {fp32,bf16} does the same for training (default fp32, the reference's arithmetic);
  * --deterministic (opt-in extension: FLAGS has no `deterministic` attribute unless it is given) trains on fixed-order
    reductions: every gradient, batch-norm and loss sum, and the gradient sum over ranks, adds in an order set by the
    shapes alone, so two runs with the same seed, data, build, GPU model and rank count give bit-identical variables,
    Adam moments, losses and outputs (the default atomic kernels agree only to rounding);
  * --outscale s (opt-in extension, absent from FLAGS unless given; inference only, 1 <= s <= 16) writes
    int(w_LR * s) x int(h_LR * s) files, Real-ESRGAN's convention: the network still runs at 4x and each output frame is
    resized on the GPU (tecogan_b200/csrc/resize.cu) to the bytes cv2.resize(frame, size, INTER_LANCZOS4) gives, before
    it is encoded; --outscale 4 writes the files of a run without the flag;
  * --input_y4m PATH / --output_y4m PATH (opt-in extensions, absent from FLAGS unless given; inference only) read the
    input from and write the output to a YUV4MPEG2 stream (8-bit 4:2:0, limited range; a file, a FIFO or /dev/stdin),
    converted on the GPU (tecogan_b200/csrc/yuv.cu) byte for byte as cv2.cvtColor(COLOR_YUV2RGB_I420 /
    COLOR_RGB2YUV_I420) converts; y4m input names its files <output_name>_<%04d frame number>.<output_ext>, y4m output
    holds the frames the image path would write and no image file is written;
  * --scene_threshold T (opt-in extension, absent from FLAGS unless given; inference only, 0 < T <= 100) restarts the
    recurrence at scene cuts: a frame whose score (the 0..100 mean absolute difference of its 8-bit RGB values to the
    previous frame's, or its change if smaller; computed on the GPU by tecogan_b200/csrc/scene.cu) is >= T starts a new
    scene, and each scene is warmed up and super-resolved as a sequence of its own, every input frame written once
    (lib/dataloader.py::scene_order; DESIGN.md section 4.13); a stream of 6 or more frames without a cut gives the files
    of a run without the flag;
  * under `torchrun` each rank trains on its own clip shard with one NCCL all-reduce per step;
  * monitoring (--summary_dir: TensorBoard scalars, logfile.txt, validation scalars, test-sequence frames at every
    checkpoint) runs on rank 0 only, in process: the held-out scenes end_dir+1..end_dir_val are optional (validation is
    skipped with a message when they are absent) and the test sequence is super-resolved synchronously instead of by an
    un-awaited subprocess.
"""
import argparse
import itertools
import math
import os
import sys
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

FLAG_DEFS = [  # (name, type, default) -- reference main.py:32-103
    ('rand_seed', int, 1), ('input_dir_LR', str, None), ('input_dir_len', int, -1), ('input_dir_HR', str, None),
    ('mode', str, 'inference'), ('output_dir', str, None), ('output_pre', str, ''), ('output_name', str, 'output'),
    ('output_ext', str, 'jpg'), ('summary_dir', str, None), ('checkpoint', str, None), ('num_resblock', int, 16),
    ('pre_trained_model', bool, False), ('vgg_ckpt', str, None), ('cudaID', str, '0'), ('queue_thread', int, 6),
    ('name_video_queue_capacity', int, 512), ('video_queue_capacity', int, 256), ('video_queue_batch', int, 2),
    ('RNN_N', int, 10), ('batch_size', int, 4), ('flip', bool, True), ('random_crop', bool, True),
    ('movingFirstFrame', bool, True), ('crop_size', int, 32), ('input_video_dir', str, ''), ('input_video_pre', str, 'scene'),
    ('str_dir', int, 1000), ('end_dir', int, 2000), ('end_dir_val', int, 2050), ('max_frm', int, 119),
    ('vgg_scaling', float, -0.002), ('warp_scaling', float, 1.0), ('pingpang', bool, False), ('pp_scaling', float, 1.0),
    ('EPS', float, 1e-12), ('learning_rate', float, 0.0001), ('decay_step', int, 500000), ('decay_rate', float, 0.5),
    ('stair', bool, False), ('beta', float, 0.9), ('adameps', float, 1e-8), ('max_epoch', int, None), ('max_iter', int, 1000000),
    ('display_freq', int, 20), ('summary_freq', int, 100), ('save_freq', int, 10000), ('ratio', float, 0.01),
    ('Dt_mergeDs', bool, True), ('Dt_ratio_0', float, 1.0), ('Dt_ratio_add', float, 0.0), ('Dt_ratio_max', float, 1.0),
    ('Dbalance', float, 0.4), ('crop_dt', float, 0.75), ('D_LAYERLOSS', bool, True),
    ('precision', str, 'bf16'),          # extension: inference arithmetic (bf16 wgmma | fp32 CUDA cores)
    ('train_precision', str, 'fp32'),    # extension: training convolutions (fp32 as the reference | bf16 wgmma)
    ('synthetic_data', bool, False),     # extension: seeded synthetic HR clips / random frozen VGG instead of raising
    # extension: fixed-order training reductions, bit-identical reruns of one seed.  Opt-in: absent from FLAGS unless
    # given (argparse.SUPPRESS), so the flag set of a run without it stays exactly the reference's.
    ('deterministic', bool, argparse.SUPPRESS),
    # extension: inference files of int(w * s) x int(h * s) instead of 4x (1 <= s <= 16), resized on the GPU as
    # cv2.resize(INTER_LANCZOS4) does.  Opt-in in the same way.
    ('outscale', float, argparse.SUPPRESS),
    # extension: inference input / output as a YUV4MPEG2 stream (tecogan_b200/y4m.py).  Opt-in in the same way.
    ('input_y4m', str, argparse.SUPPRESS), ('output_y4m', str, argparse.SUPPRESS),
    # extension: restart the inference recurrence at scene cuts (score >= T, 0 < T <= 100).  Opt-in in the same way;
    # read as text and checked by main(), so that a malformed value raises ValueError as an out-of-range one does.
    ('scene_threshold', str, argparse.SUPPRESS),
]


def parse_flags(argv=None):
    """tf.app.flags-style parsing: `--name value`, `--name=value`, booleans as `--name` / `--noname`."""
    ap = argparse.ArgumentParser(allow_abbrev=False)
    for name, typ, default in FLAG_DEFS:
        if typ is bool:
            ap.add_argument('--' + name, dest=name, nargs='?', const=True, default=default,
                            type=lambda s: s.lower() in ('1', 'true', 'yes'))
            ap.add_argument('--no' + name, dest=name, action='store_false', default=default)
        else:
            ap.add_argument('--' + name, type=typ, default=default)
    return ap.parse_args(argv)


def load_checkpoint(store, spec, num_resblock, need_d=False, need_vgg=False, pre_trained_model=False, vgg_ckpt=None):
    """--checkpoint: `random:<seed>`, a .pt file written by this main.py, or a TensorFlow checkpoint (V2 prefix such as
    ./model/TecoGAN, or a V1 file) read without TensorFlow by tecogan_b200/tf_bundle.py.

    TF checkpoints follow the reference: inference restores the generator + fnet variables and fails on a missing one
    (Saver.restore, main.py:221-224,245); training with --pre_trained_model loads what exists, zero-fills missing
    generator/fnet variables and leaves missing discriminator variables at their initial values (main.py:312-320,
    lib/ops.py:370-391); without it everything must be present (main.py:346-349; optimiser state follows in
    restore_train_state once the trainer exists).  --vgg_ckpt is read the same way (main.py:322-343)."""
    import torch
    from tecogan_b200 import tf_bundle
    from tecogan_b200.init_params import variable_shapes, xavier_params
    if spec.startswith('random:'):
        store.load(xavier_params(int(spec.split(':', 1)[1]), num_resblock, need_d, need_vgg))
    elif tf_bundle.is_tf_checkpoint(spec):
        reader = tf_bundle.load_checkpoint(spec)
        shapes = variable_shapes(num_resblock, need_d, False)
        gen_fnet = {k: v for k, v in shapes.items() if not k.startswith('tdiscriminator/')}
        dis = {k: v for k, v in shapes.items() if k.startswith('tdiscriminator/')}
        if pre_trained_model:
            got = tf_bundle.get_existing_from_ckpt(reader, gen_fnet, rest_zero=True, print_level=1)
            print('Prepare to load %d weights from the pre-trained model for generator and fnet' % len(got))
            dgot = tf_bundle.get_existing_from_ckpt(reader, dis, print_level=0)
            if dis:
                print('Prepare to load %d weights from the pre-trained model for discriminator' % len(dgot))
            got.update(dgot)
        else:
            missing = [k for k in shapes if not reader.has_tensor(k)]
            if missing:
                raise ValueError('checkpoint %s lacks %d variables of this graph, e.g. %s' % (spec, len(missing), missing[:3]))
            got = tf_bundle.get_existing_from_ckpt(reader, shapes, print_level=0)
        reader.close()
        store.load({k: torch.from_numpy(v) for k, v in got.items()})
    else:
        blob = torch.load(spec, map_location='cpu')      # variables only: optimiser slots / counters go through restore_train_state
        blob = {k: v for k, v in blob.items() if not (k.endswith('/Adam') or k.endswith('/Adam_1') or k == 'global_step'
                                                      or k.startswith('teco_b200/'))}
        # same strictness as Saver.restore / the TF branch above: every variable of this graph, with the right shape
        shapes = variable_shapes(num_resblock, need_d, False)
        for k, shp in shapes.items():
            if k in blob and tuple(blob[k].shape) != tuple(shp):
                raise ValueError('Wrong shape in for {} in ckpt,expected {}, got {}.'.format(k, str(tuple(shp)), str(tuple(blob[k].shape))))
        missing = [k for k in shapes if k not in blob]
        if missing and pre_trained_model:   # lib/ops.py:370-391: generator/fnet variables absent from the file are zero-filled
            for k in missing:
                if not k.startswith('tdiscriminator/'):
                    blob[k] = torch.zeros(shapes[k])
            print('Prepare to load %d weights from the pre-trained model (%d not in the file)' % (len(blob), len(missing)))
        elif missing:
            raise ValueError('checkpoint %s lacks %d variables of this graph (num_resblock=%d%s), e.g. %s'
                             % (spec, len(missing), num_resblock, ', discriminator' if need_d else '', missing[:3]))
        store.load(blob)
    if need_vgg and vgg_ckpt is not None:
        load_vgg_checkpoint(store, vgg_ckpt)


def load_vgg_checkpoint(store, vgg_ckpt):
    """--vgg_ckpt (slim's vgg_19.ckpt, a V1 checkpoint): the 16 convolutions of vgg_19 (reference main.py:322-324,340-343)."""
    import torch
    from tecogan_b200 import tf_bundle
    from tecogan_b200.init_params import variable_shapes
    reader = tf_bundle.load_checkpoint(vgg_ckpt)
    vshapes = {k: v for k, v in variable_shapes(1, False, True).items() if k.startswith('vgg_19/')}
    missing = [k for k in vshapes if not reader.has_tensor(k)]
    if missing:
        raise ValueError('vgg checkpoint %s lacks %s' % (vgg_ckpt, missing[:3]))
    store.load({k: torch.from_numpy(v) for k, v in tf_bundle.get_existing_from_ckpt(reader, vshapes, print_level=0).items()})
    reader.close()
    print('VGG19 restored successfully!!')


def save_checkpoint(store, output_dir, step, train_state=None):
    """Both a .pt file and a TensorFlow V2 bundle `model-<step>.{index,data-00000-of-00001}` (Saver.save naming,
    main.py:362-366,418-421) holding every variable under its TF name, `global_step`, and -- when the trainer is given --
    the Adam moments under TF's slot names plus the step counters / EMAs needed for an exact resume."""
    import numpy as np
    import torch
    from tecogan_b200 import tf_bundle
    params = {k: v.detach().cpu() for k, v in store.items()}
    params['global_step'] = torch.tensor(step, dtype=torch.int64)
    if train_state is not None:
        params.update(train_state.state_tensors())
    torch.save(params, os.path.join(output_dir, 'model-%d.pt' % step))
    tf_bundle.write_bundle(os.path.join(output_dir, 'model-%d' % step), {k: np.asarray(v.numpy()) for k, v in params.items()})


def restore_train_state(train_state, spec):
    """Continue a training run (reference main.py:346-349 "Loading everything from the checkpoint"): optimiser moments,
    global_step and the EMAs from a checkpoint written by save_checkpoint, or -- for a TensorFlow checkpoint of the
    reference -- the Adam slots it holds (found by name suffix) and global_step."""
    import torch
    from tecogan_b200 import tf_bundle
    if spec.startswith('random:'):
        return []
    if tf_bundle.is_tf_checkpoint(spec):
        reader = tf_bundle.load_checkpoint(spec)
        keys = reader.keys()

        def get(name):
            if reader.has_tensor(name):
                return reader.get_tensor(name)
            if name.endswith('/Adam') or name.endswith('/Adam_1'):
                hits = [k for k in keys if k.endswith('/' + name)]
                if len(hits) == 1:
                    return reader.get_tensor(hits[0])
            return None
        missing = train_state.load_state(get)
        reader.close()
    else:
        blob = torch.load(spec, map_location='cpu')
        missing = train_state.load_state(lambda name: blob.get(name))
    if missing:
        print('[main] resume: %d state entries not in the checkpoint (kept at their initial values), e.g. %s' % (len(missing), missing[:3]))
    return missing


def inference(FLAGS):
    from tecogan_b200 import config, variables as V, y4m
    from tecogan_b200.engine import InferenceEngine
    from tecogan_b200.lib.dataloader import inference_paths, padded, stream_inputs, stream_scenes
    if FLAGS.checkpoint is None:
        raise ValueError('The checkpoint file is needed to performing the test.')
    sink = None
    scenes = hasattr(FLAGS, 'scene_threshold')
    if hasattr(FLAGS, 'input_y4m'):            # the header is read and checked here, before anything is set up
        reader = y4m.Y4MReader(FLAGS.input_y4m, FLAGS.input_dir_len)
        rate, aspect = reader.header.rate, reader.header.aspect
        if scenes:
            frames, names = reader.scenes(FLAGS.scene_threshold), reader.name
        else:
            frames, names = reader.frames(), reader.names()
    else:
        paths, down = inference_paths(FLAGS)
        rate, aspect = y4m.PNG_INPUT_RATE, y4m.PNG_INPUT_ASPECT
        if scenes:
            frames, names = stream_scenes(paths, down, FLAGS.scene_threshold), paths.__getitem__
        else:
            frames, names = stream_inputs(paths, down), padded(paths)
    try:
        first = next(frames, None)
        if first is None:
            raise IndexError('no frame in the input y4m stream' if hasattr(FLAGS, 'input_y4m')
                             else 'no .png frame in the input directory')
        h, w = (first.frame if scenes else first).shape[:2]
        out_hw = outscale_size(FLAGS, h, w)
        if hasattr(FLAGS, 'output_y4m') and (out_hw[0] % 2 or out_hw[1] % 2):
            raise ValueError('--output_y4m: the %dx%d output has an odd side; 4:2:0 needs even sides (choose another '
                             '--outscale)' % (out_hw[1], out_hw[0]))
        print("input shape:", [1, h, w, 3])
        print("output shape:", [1] + list(out_hw) + [3])
        config.set_precision(FLAGS.precision)
        store = V.set_default_store(V.VariableStore(seed=FLAGS.rand_seed))
        load_checkpoint(store, FLAGS.checkpoint, FLAGS.num_resblock)
        eng = InferenceEngine(h, w, FLAGS.num_resblock)
        print('Finish building the network')
        image_dir = FLAGS.output_dir if FLAGS.output_pre == "" else os.path.join(FLAGS.output_dir, FLAGS.output_pre)
        if hasattr(FLAGS, 'output_y4m'):
            sink = y4m.Y4MWriter(FLAGS.output_y4m, out_hw[1], out_hw[0], rate, aspect)
        else:
            os.makedirs(image_dir, exist_ok=True)
        run = super_resolve_scenes if scenes else super_resolve_frames
        run(eng, names, itertools.chain([first], frames), image_dir, FLAGS.output_name, FLAGS.output_ext, out_hw, sink)
    finally:
        frames.close()
        if sink is not None:
            sink.close()


def outscale_size(FLAGS, h, w):
    """(height, width) of the files inference writes for an h x w input: 4x, or with --outscale s
    (int(h * s), int(w * s))."""
    from tecogan_b200 import resize
    if not hasattr(FLAGS, 'outscale'):
        return 4 * h, 4 * w
    resize.check_outscale(FLAGS.outscale)
    return resize.out_size(h, w, FLAGS.outscale)


def super_resolve_frames(eng, paths_LR, frames, image_dir, output_name, output_ext, out_hw=None, sink=None):
    """The per-frame loop of reference main.py:253-268: every frame through `eng`, the 5 warm-up frames discarded, the
    rest saved as <output_name>_<frame name>.<output_ext>.  paths_LR is the padded file list and `frames` its [h, w, 3]
    float32 frames in the same order (lib/dataloader.py::stream_inputs: decoded a window ahead on a reader thread).
    The loop runs to the end of `frames`, whose length need not be known; paths_LR may be any iterable of paths or
    names taken in step with it (tecogan_b200/y4m.py::Y4MReader.names for --input_y4m).  With a `sink`
    (y4m.Y4MWriter, --output_y4m) the frames that would be saved are appended to it instead, and no file is written.

    The host does not wait for the device: each step's next frame is already on its way when the step is enqueued
    (its flow is estimated while this frame is generated), and each output frame is copied to a FrameWriter slot,
    encoded and written behind the steps that follow.  The files and the printed lines are those of the serial loop;
    "total time" is the sum of the steps' device times (CUDA events around each step).  `out_hw` (--outscale) is the
    files' (height, width) when it is not the network's 4x: the writer resizes each frame to it on the device
    (lib/writer.py::FrameWriter)."""
    import collections
    import torch
    from tecogan_b200.lib.writer import FrameWriter
    it, names = iter(frames), iter(paths_LR)
    max_iter = 0
    srtime = 0.0
    timing = collections.deque()           # (start, end) events of steps whose time is not yet counted
    writer = None
    print('Frame evaluation starts!!')
    try:
        cur = next(it, None)
        for i in itertools.count():
            if cur is None:
                break
            path = next(names)
            nxt = next(it, None)
            t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            t0.record()
            eng.step(cur, next_lr=nxt)
            t1.record()
            timing.append((t0, t1))
            while timing and timing[0][1].query():
                a, b = timing.popleft()
                srtime += a.elapsed_time(b) / 1000.0
            cur = nxt
            max_iter = i + 1
            if i >= 5:
                name, _ = os.path.splitext(os.path.basename(str(path)))
                filename = output_name + '_' + name
                print('saving image %s' % filename)
                if writer is None:
                    writer = FrameWriter(*(out_hw or eng.out_u8.shape[1:3]), eng.device, sink=sink)
                writer.put(eng.out_u8[0], os.path.join(image_dir, "%s.%s" % (filename, output_ext)))
            else:   # First 5 is a hard-coded symmetric frame padding, ignored but time added!
                print("Warming up %d" % (5 - i))
        cur = nxt = None
    finally:
        if writer is not None:
            writer.close()
    if writer is not None and writer.error is not None:
        raise writer.error
    torch.cuda.synchronize()
    for a, b in timing:
        srtime += a.elapsed_time(b) / 1000.0
    print("total time " + str(srtime) + ", frame number " + str(max_iter))


def super_resolve_scenes(eng, name_of, steps, image_dir, output_name, output_ext, out_hw=None, sink=None):
    """super_resolve_frames for a stream cut into scenes (--scene_threshold): `steps` are the
    lib/dataloader.py::SceneSteps of stream_scenes or Y4MReader.scenes.  Before a scene's first step the engine is reset
    (pre_warp = 0) and, for a scene that starts at a cut, `scene cut before frame <i>, score <s>` is printed; its
    warm-up steps print `Warming up <n>` and are not saved; each written step saves its frame as
    <output_name>_<name>.<output_ext>, name_of(input index) giving the name (a path's stem, or y4m's %04d).  The next
    frame's flow is computed ahead (step(cur, next_lr=nxt)) except across a scene boundary: a scene's last frame is
    stepped alone, then the engine is reset.  "frame number" counts every step, warm-ups included.  Writing, timing and
    errors are as in super_resolve_frames."""
    import collections
    import torch
    from tecogan_b200.lib.writer import FrameWriter
    it = iter(steps)
    steps_run = 0
    srtime = 0.0
    timing = collections.deque()
    writer = None
    warm = 0
    print('Frame evaluation starts!!')
    try:
        cur = next(it, None)
        while cur is not None:
            nxt = next(it, None)
            if cur.reset:
                if cur.score is not None:
                    print('scene cut before frame %d, score %.4f' % (cur.start, cur.score))
                eng.reset()
                warm = cur.index - cur.start
            t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            t0.record()
            eng.step(cur.frame, next_lr=nxt.frame if nxt is not None and not nxt.reset else None)
            t1.record()
            timing.append((t0, t1))
            while timing and timing[0][1].query():
                a, b = timing.popleft()
                srtime += a.elapsed_time(b) / 1000.0
            steps_run += 1
            if cur.write:
                name, _ = os.path.splitext(os.path.basename(str(name_of(cur.index))))
                filename = output_name + '_' + name
                print('saving image %s' % filename)
                if writer is None:
                    writer = FrameWriter(*(out_hw or eng.out_u8.shape[1:3]), eng.device, sink=sink)
                writer.put(eng.out_u8[0], os.path.join(image_dir, "%s.%s" % (filename, output_ext)))
            else:
                print("Warming up %d" % warm)
                warm -= 1
            cur = nxt
        cur = nxt = None
    finally:
        if writer is not None:
            writer.close()
    if writer is not None and writer.error is not None:
        raise writer.error
    torch.cuda.synchronize()
    for a, b in timing:
        srtime += a.elapsed_time(b) / 1000.0
    print("total time " + str(srtime) + ", frame number " + str(steps_run))


TEST_SEQUENCE_DIR = './LR/calendar/'      # reference main.py:164, hard-coded there as well


def synthetic_hr_batch(FLAGS, step, rank, device, validation=False):
    """Seeded smooth-noise HR clips [B,RNN_N,4crop+8,4crop+8,3] in [0,1] moving by a constant sub-pixel velocity.
    Training batch `step` of `rank` uses seed 1000003 * rank + step; validation batch `step` counts down from the top of
    the generator's 32-bit seed range, which no training batch reaches (fewer than 4000 ranks, 4e9 steps)."""
    import torch
    g = torch.Generator().manual_seed(0xFFFFFFFF - step if validation else 1000003 * rank + step)
    B, T, S = FLAGS.batch_size, FLAGS.RNN_N, FLAGS.crop_size * 4 + 8
    base = torch.rand(B, 3, S // 8 + 8, S // 8 + 8, generator=g)
    big = torch.nn.functional.interpolate(base, scale_factor=8, mode='bicubic', align_corners=False).clamp(0, 1)
    out = torch.empty(B, T, S, S, 3)
    for t in range(T):
        oy, ox = 8 + 2 * t, 8 + t
        out[:, t] = big[:, :, oy:oy + S, ox:ox + S].permute(0, 2, 3, 1)
    return out.to(device)


def test_while_train(FLAGS, step):
    """reference main.py:151-174 (testWhileTrain), in process and synchronous: the first 10 frames of ./LR/calendar/
    super-resolved with the current weights at the --precision inference arithmetic into <output_dir>/train/ as
    <%09d step>_<frame>.<output_ext> -- the files `main.py --mode inference --input_dir_len 10 --output_name %09d
    --output_pre ""` writes.  The global precision is restored and the engine (its CUDA graph, buffers and packed weights)
    is released before training continues; the training step keeps its own buffers and repacks its weights."""
    import argparse
    import torch
    from tecogan_b200 import config
    from tecogan_b200.engine import InferenceEngine
    from tecogan_b200.lib.dataloader import inference_paths, padded, stream_inputs
    print('[testWhileTrain] step %d:' % step)
    if not os.path.isdir(TEST_SEQUENCE_DIR):
        print('[testWhileTrain] %s not found, no test-sequence frames' % TEST_SEQUENCE_DIR)
        return
    tflags = argparse.Namespace(input_dir_LR=TEST_SEQUENCE_DIR, input_dir_HR=None, input_dir_len=10)
    paths, down = inference_paths(tflags)
    image_dir = os.path.join(FLAGS.output_dir, 'train')
    os.makedirs(image_dir, exist_ok=True)
    prev_precision = config.precision()
    frames = stream_inputs(paths, down)
    eng = None
    try:
        first = next(frames, None)
        if first is None:
            raise IndexError('no .png frame in ' + TEST_SEQUENCE_DIR)
        config.set_precision(FLAGS.precision)
        eng = InferenceEngine(first.shape[0], first.shape[1], FLAGS.num_resblock)
        super_resolve_frames(eng, padded(paths), itertools.chain([first], frames), image_dir, '%09d' % step,
                             FLAGS.output_ext)
    finally:
        frames.close()                    # the reader thread is joined, the writer was joined by super_resolve_frames
        first = eng = None
        torch.cuda.synchronize()
        config.set_precision(prev_precision)


def validation_source(FLAGS, dev):
    """k -> HR validation batch k (reference lib/dataloader.py:287-297), or None when there is no validation data.
    Batch k depends on k only, so a resumed run sees the same validation batches."""
    if FLAGS.input_video_dir:
        from tecogan_b200.lib.dataloader import validation_loader
        loader, why = validation_loader(FLAGS)
        if loader is None:
            print('[main] validation skipped: %s' % why)
            return None

        def fetch(k):
            return loader.batch(k).to(dev)
        fetch.loader = loader               # train() moves validation onto the frame store with it
        return fetch
    return lambda k: synthetic_hr_batch(FLAGS, k, 0, dev, validation=True)


def frame_store_fits(store_bytes, free_bytes, reserved_bytes, peak_bytes, total_bytes, host_room_bytes=None):
    """Where the frame store (lib/dataloader.py::FrameStore) fits beside training: (placement, message).

    The reserve is a measured peak.  train() decides after the first training step, after the test-sequence pass (at the
    start, with --summary_dir) and after one validation pass, so `peak_bytes` (torch.cuda.max_memory_allocated) is the most
    those passes and the model have held at once.  The process can use `free_bytes` (cudaMemGetInfo) plus what PyTorch's
    allocator has reserved (`reserved_bytes`); the store fits when it leaves the peak and a margin of max(1 GiB, 5 % of the
    device's `total_bytes`) -- allocator fragmentation, NCCL and library workspaces -- inside that.

    Without `host_room_bytes` the placement is True (the device) or False, as it always was.  With it (the bytes of host
    memory the node can give the store, tecogan_b200/hostmem.py::host_room_bytes) the placement is 'device' when the
    store fits on the device, else 'host' when it fits in `host_room_bytes`, else False (the host loader)."""
    margin = max(1 << 30, total_bytes // 20)
    room = free_bytes + reserved_bytes - peak_bytes - margin
    gib = lambda b: b / float(1 << 30)
    fits = store_bytes <= room
    msg = ('frame store %.2f GiB %s the %.2f GiB left beside a measured peak of %.2f GiB and a %.2f GiB margin'
           % (gib(store_bytes), 'fits in' if fits else 'does not fit in', gib(max(room, 0)), gib(peak_bytes), gib(margin)))
    if host_room_bytes is None:
        return fits, msg
    if fits:
        return 'device', msg
    host = store_bytes <= host_room_bytes
    msg += ', and %s the %.2f GiB of host memory left beside the host margin' % ('fits in' if host else 'does not fit in',
                                                                                 gib(max(host_room_bytes, 0)))
    return ('host' if host else False), msg


PLACEMENT_CODES = {'device': 2, 'host': 1}         # ranks agree on the smallest; 0 is the host loader


def node_host_room(rank, world):
    """host_room_bytes() as measured by the lowest rank on this rank's host (one host store serves all of them)."""
    from tecogan_b200.hostmem import host_room_bytes, node_groups
    if world <= 1:
        return host_room_bytes()
    import socket
    import torch.distributed as dist
    got = [None] * world
    dist.all_gather_object(got, (socket.gethostname(), host_room_bytes()))
    return got[node_groups([h for h, _ in got])[rank][0]][1]


def select_training_input(FLAGS, Net, loader, val_hr, batch, next_step, dev, rank, world, monitor):
    """After the first training step from disk: read the training (and validation) clips from a FrameStore on the device
    when it fits, else from a FrameStore in host memory when that fits (frame_store_fits; under torchrun every rank takes
    the smallest placement of any rank), otherwise -- or when the host memory cannot be set up (created, shared or
    registered with the device) -- from the host loader's thread pool.  Either way the batches are the same, bit for bit.  Returns (next_hr, val_hr)."""
    import torch
    import torch.distributed as dist
    from tecogan_b200.hostmem import HostStoreError
    from tecogan_b200.lib.dataloader import FrameStore, validation_loader
    val_loader = None
    if monitor and val_hr is not None:
        val_loader = val_hr.loader
        Net.train.evaluate(*batch)        # the validation pass's allocations count in the peak (nothing is written)
    elif FLAGS.summary_dir and not monitor:
        val_loader = validation_loader(FLAGS)[0]     # rank 0 validates: every rank stores the same scenes
    loaders = [loader] + ([val_loader] if val_loader is not None else [])
    torch.cuda.synchronize()
    store_bytes = FrameStore.estimate_bytes(loaders)
    free, total = torch.cuda.mem_get_info(dev)
    placement, msg = frame_store_fits(store_bytes, free, torch.cuda.memory_reserved(dev),
                                      torch.cuda.max_memory_allocated(dev), total, node_host_room(rank, world))
    code = PLACEMENT_CODES.get(placement, 0)
    if world > 1:
        agree = torch.tensor([code], dtype=torch.int32, device=dev)
        dist.all_reduce(agree, op=dist.ReduceOp.MIN)
        if agree.item() < code:
            msg += ' on this rank, not on every rank'
        code = int(agree.item())
    placement = {v: k for k, v in PLACEMENT_CODES.items()}.get(code)
    host_loader = 'host loader (%d threads)' % loader.queue_thread
    if rank == 0:
        print('[main] %s: training reads its clips from the %s' % (msg, {'device': 'frame store on the device',
                                                                         'host': 'frame store in host memory'}.get(
                                                                             placement, host_loader)))
    store = None
    if placement == 'host':
        try:
            store = FrameStore(loaders, dev, rank=rank, world=world, placement='host')
        except HostStoreError as e:
            if rank == 0:
                print('[main] %s: training reads its clips from the %s' % (e, host_loader))
    elif placement == 'device':
        store = FrameStore(loaders, dev, rank=rank, world=world)
    if store is None:
        clip_iter = loader.batches(start_step=next_step)
        return (lambda gstep: next(clip_iter).to(dev, non_blocking=True)), val_hr
    if rank == 0:
        print('[main] frame store: %d frames, %.2f GiB, built in %.1f s' % (len(store.paths), store.nbytes / float(1 << 30),
                                                                           store.build_seconds))
    clip_iter = store.batches(start_step=next_step)
    if val_loader is not None and val_hr is not None:
        vstore = store.view(val_loader)

        def fetch(k):
            return vstore.batch(k)
        fetch.loader = val_loader
        val_hr = fetch
    return (lambda gstep: next(clip_iter)), val_hr


def train(FLAGS):
    if not FLAGS.input_video_dir and not FLAGS.synthetic_data:
        raise ValueError('Video input directory input_video_dir is not provided')       # reference lib/dataloader.py:159-160
    if FLAGS.vgg_scaling > 0 and FLAGS.vgg_ckpt is None and not FLAGS.synthetic_data:
        raise ValueError('vgg_scaling > 0 needs --vgg_ckpt (the reference always restores vgg_19.ckpt, main.py:322-343); '
                         'pass --synthetic_data to run on a seeded random frozen VGG')
    import torch
    import torch.distributed as dist
    from tecogan_b200 import variables as V
    from tecogan_b200.lib.dataloader import frvsr_gpu_data_loader
    from tecogan_b200.lib.Teco import FRVSR, TecoGAN
    rank, world = int(os.environ.get('RANK', '0')), int(os.environ.get('WORLD_SIZE', '1'))
    local_rank = int(os.environ.get('LOCAL_RANK', '0'))
    torch.cuda.set_device(local_rank)
    if world > 1:
        dist.init_process_group('nccl', device_id=torch.device('cuda', local_rank))
    from tecogan_b200 import config
    config.set_train_precision(FLAGS.train_precision)   # fp32 as the reference; bf16: wgmma convolutions, fp32 master weights
    config.set_deterministic(getattr(FLAGS, 'deterministic', False))
    store = V.set_default_store(V.VariableStore(seed=FLAGS.rand_seed))   # same seed on every rank -> identical init
    gan = FLAGS.ratio > 0
    if FLAGS.checkpoint is not None:
        load_checkpoint(store, FLAGS.checkpoint, FLAGS.num_resblock, gan, FLAGS.vgg_scaling > 0,
                        pre_trained_model=FLAGS.pre_trained_model, vgg_ckpt=FLAGS.vgg_ckpt)
    elif FLAGS.vgg_scaling > 0 and FLAGS.vgg_ckpt is not None:
        load_vgg_checkpoint(store, FLAGS.vgg_ckpt)
    elif FLAGS.vgg_scaling > 0:
        print('[main] --synthetic_data: VGG19 uses seeded random weights (frozen) -- the perceptual loss is NOT the reference\'s')
    dev = torch.device('cuda', local_rank)
    if FLAGS.input_video_dir:
        # HR clips from disk (reference lib/dataloader.py:147-273): decoded + augmented on queue_thread host threads,
        # uploaded from pinned memory; LR synthesis and target crops happen on the device (frvsr_gpu_data_loader)
        from tecogan_b200.lib.dataloader import HRClipLoader
        loader = HRClipLoader(FLAGS, rank=rank, world=world)
        if FLAGS.max_iter is None:            # reference main.py:370-375
            if FLAGS.max_epoch is None:
                raise ValueError('one of max_epoch or max_iter should be provided')
            FLAGS.max_iter = FLAGS.max_epoch * loader.steps_per_epoch
    else:
        loader = None
    # the graph is built on a shape-only batch (its values are never trained on); the data stream starts afterwards, at
    # the restored global step, so a resumed run sees exactly the batches the uninterrupted run would have seen
    B_, T_, S_ = FLAGS.batch_size, FLAGS.RNN_N, FLAGS.crop_size * 4 + 8
    lr0, tg0 = frvsr_gpu_data_loader(torch.zeros((B_, T_, S_, S_, 3), device=dev), FLAGS)
    Net = TecoGAN(lr0, tg0, FLAGS) if gan else FRVSR(lr0, tg0, FLAGS)
    print('Finish building the network.')
    if FLAGS.checkpoint is not None and not FLAGS.pre_trained_model:
        print('Loading everything from the checkpoint to continue the training...')
        restore_train_state(Net.train, FLAGS.checkpoint)
    start_step = Net.global_step()
    monitor = bool(FLAGS.summary_dir) and rank == 0      # summaries, validation, test sequence: rank 0, no collective
    if monitor:
        from tecogan_b200.summary import EventWriter
        writer = EventWriter(FLAGS.summary_dir)
        # the GIF summaries go to a sibling run: readers of the scalar file see only simple values
        gif_writer = EventWriter(os.path.join(FLAGS.summary_dir, 'gif'))
        val_hr = validation_source(FLAGS, dev)
        test_while_train(FLAGS, start_step)
    tested = {start_step}
    if loader is not None:
        # the first step's batch is decoded on this thread; after that step select_training_input moves the input to
        # the device frame store when it fits, or to the host loader's thread pool
        next_hr = lambda gstep: loader.batch(gstep).to(dev, non_blocking=True)
    else:
        next_hr = lambda gstep: synthetic_hr_batch(FLAGS, gstep, rank, dev)   # seeded by the GLOBAL step
    frame_len = (FLAGS.RNN_N * 2 - 1) if FLAGS.pingpang else FLAGS.RNN_N
    max_iter, start = FLAGS.max_iter, time.time()
    try:
        for step in range(max(0, max_iter - start_step)):
            lr_, tg_ = frvsr_gpu_data_loader(next_hr(start_step + step), FLAGS)
            res = Net.train(lr_, tg_)
            run_step = Net.global_step()
            if step == 0 and rank == 0:
                print('Optimization starts!!!(Ctrl+C to stop, will try saving the last model...)')
            if monitor and (run_step % FLAGS.summary_freq) == 0:     # reference main.py:384-402
                print('Run and Recording summary!!')
                writer.add_scalars(run_step, [('learning_rate', res["lr"])] + list(zip(Net.update_list_name, Net.update_list_avg())))
                gif_writer.add_images(run_step, Net.image_summary())
                if val_hr is not None:
                    val = Net.train.evaluate(*frvsr_gpu_data_loader(val_hr(run_step // FLAGS.summary_freq), FLAGS))
                    writer.add_scalars(run_step, [('val_' + name, v) for name, v in val.items()])
                    print('-----------Validation data scalars-----------')
                    for name, v in val.items():
                        print('val_' + name, v)
            if (run_step % FLAGS.display_freq) == 0 and rank == 0:
                rate = (step + 1) * FLAGS.batch_size * world / (time.time() - start)
                remaining = (max_iter - start_step - step) * FLAGS.batch_size * world / rate
                print("progress  step %d  image/sec %0.1fx%02d  remaining %dh%dm" %
                      (run_step, rate, frame_len, remaining // 3600, (remaining % 3600) // 60))
                print("global_step", run_step)
                print("learning_rate", res["lr"])
                for name, value in zip(Net.update_list_name, Net.update_list_avg()):
                    print(name, value)
            if (run_step % FLAGS.save_freq) == 0 and rank == 0:
                print('Save the checkpoint')
                save_checkpoint(store, FLAGS.output_dir, run_step, Net.train)
                if monitor:
                    test_while_train(FLAGS, run_step)
                    tested.add(run_step)
            if step == 0 and loader is not None:
                next_hr, val_hr = select_training_input(FLAGS, Net, loader, val_hr if monitor else None, (lr_, tg_),
                                                        start_step + 1, dev, rank, world, monitor)
    except KeyboardInterrupt:
        if rank == 0:
            print('main.py: KeyboardInterrupt->saving the checkpoint')
            save_checkpoint(store, FLAGS.output_dir, Net.global_step(), Net.train)
            if monitor:
                test_while_train(FLAGS, Net.global_step())
        print('main.py: quit')
        sys.exit(0)
    if rank == 0:
        save_checkpoint(store, FLAGS.output_dir, Net.global_step(), Net.train)
        if monitor and Net.global_step() not in tested:
            test_while_train(FLAGS, Net.global_step())
    if monitor:
        writer.close()
        gif_writer.close()
    print('Optimization done!!!!!!!!!!!!')
    if world > 1:
        dist.destroy_process_group()


def main(argv=None):
    FLAGS = parse_flags(argv)
    for flag in ('input_y4m', 'output_y4m'):    # refused before anything is set up
        if hasattr(FLAGS, flag) and FLAGS.mode != 'inference':
            raise ValueError('--%s applies to --mode inference only' % flag)
    if hasattr(FLAGS, 'input_y4m') and (FLAGS.input_dir_LR is not None or FLAGS.input_dir_HR is not None):
        raise ValueError('--input_y4m replaces --input_dir_LR / --input_dir_HR: give one input')
    if hasattr(FLAGS, 'scene_threshold'):      # refused before anything is set up
        if FLAGS.mode != 'inference':
            raise ValueError('--scene_threshold applies to --mode inference only')
        from tecogan_b200.lib.dataloader import scene_threshold
        FLAGS.scene_threshold = scene_threshold(FLAGS.scene_threshold)
    if hasattr(FLAGS, 'outscale'):             # refused before anything is set up
        if FLAGS.mode != 'inference':
            raise ValueError('--outscale applies to --mode inference only')
        from tecogan_b200.resize import check_outscale
        check_outscale(FLAGS.outscale)
    if 'LOCAL_RANK' not in os.environ:
        os.environ["CUDA_VISIBLE_DEVICES"] = FLAGS.cudaID       # reference main.py:107: overwritten unconditionally
    if FLAGS.output_dir is None:
        raise ValueError('The output directory is needed')
    os.makedirs(FLAGS.output_dir, exist_ok=True)
    tee = None
    if FLAGS.summary_dir:
        os.makedirs(FLAGS.summary_dir, exist_ok=True)
        if os.environ.get('RANK', '0') == '0':          # reference main.py:126-136: stdout also goes to logfile.txt
            from tecogan_b200.summary import Tee
            tee = sys.stdout = Tee(os.path.join(FLAGS.summary_dir, 'logfile.txt'))
    try:
        if FLAGS.mode == 'inference':
            inference(FLAGS)
        elif FLAGS.mode == 'train':
            train(FLAGS)
        else:
            raise ValueError("mode must be 'inference' or 'train'")
    finally:
        if tee is not None:
            sys.stdout = tee.terminal
            tee.close()


if __name__ == '__main__':
    main()
