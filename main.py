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
    down-sampling, crops) is the same either way;
  * --precision {bf16,fp32} selects wgmma tensor-core or fp32 CUDA-core convolutions for inference;
    --train_precision {fp32,bf16} does the same for training (default fp32, the reference's arithmetic);
  * under `torchrun` each rank trains on its own clip shard with one NCCL all-reduce per step.
"""
import argparse
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
]


def parse_flags(argv=None):
    """tf.app.flags-style parsing: `--name value`, `--name=value`, booleans as `--name` / `--noname`."""
    ap = argparse.ArgumentParser(allow_abbrev=False)
    for name, typ, default in FLAG_DEFS:
        if typ is bool:
            ap.add_argument('--' + name, dest=name, nargs='?', const=True, default=default,
                            type=lambda s: s.lower() in ('1', 'true', 'yes'))
            ap.add_argument('--no' + name, dest=name, action='store_false')
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
    import numpy as np
    import torch
    from tecogan_b200 import config, variables as V
    from tecogan_b200.engine import InferenceEngine
    from tecogan_b200.lib.dataloader import inference_data_loader
    from tecogan_b200.lib.ops import save_img
    if FLAGS.checkpoint is None:
        raise ValueError('The checkpoint file is needed to performing the test.')
    inference_data = inference_data_loader(FLAGS)
    h, w = inference_data.inputs[0].shape[:2]
    print("input shape:", [1, h, w, 3])
    print("output shape:", [1, h * 4, w * 4, 3])
    config.set_precision(FLAGS.precision)
    store = V.set_default_store(V.VariableStore(seed=FLAGS.rand_seed))
    load_checkpoint(store, FLAGS.checkpoint, FLAGS.num_resblock)
    eng = InferenceEngine(h, w, FLAGS.num_resblock)
    print('Finish building the network')
    image_dir = FLAGS.output_dir if FLAGS.output_pre == "" else os.path.join(FLAGS.output_dir, FLAGS.output_pre)
    os.makedirs(image_dir, exist_ok=True)
    max_iter = len(inference_data.inputs)
    srtime = 0
    print('Frame evaluation starts!!')
    to_dev = lambda k: torch.from_numpy(np.array([inference_data.inputs[k]]).astype(np.float32)).cuda()
    nxt = to_dev(0)
    for i in range(max_iter):
        input_im, nxt = nxt, (to_dev(i + 1) if i + 1 < max_iter else None)
        t0 = time.time()
        out = eng.step(input_im, next_lr=nxt)     # the next frame's flow is estimated while this frame is generated
        torch.cuda.synchronize()
        srtime += time.time() - t0
        if i >= 5:
            name, _ = os.path.splitext(os.path.basename(str(inference_data.paths_LR[i])))
            filename = FLAGS.output_name + '_' + name
            print('saving image %s' % filename)
            save_img(os.path.join(image_dir, "%s.%s" % (filename, FLAGS.output_ext)), out[0])
        else:   # First 5 is a hard-coded symmetric frame padding, ignored but time added!
            print("Warming up %d" % (5 - i))
    print("total time " + str(srtime) + ", frame number " + str(max_iter))


def synthetic_hr_batch(FLAGS, step, rank, device):
    """Seeded smooth-noise HR clips [B,RNN_N,4crop+8,4crop+8,3] in [0,1] moving by a constant sub-pixel velocity."""
    import torch
    g = torch.Generator().manual_seed(1000003 * rank + step)
    B, T, S = FLAGS.batch_size, FLAGS.RNN_N, FLAGS.crop_size * 4 + 8
    base = torch.rand(B, 3, S // 8 + 8, S // 8 + 8, generator=g)
    big = torch.nn.functional.interpolate(base, scale_factor=8, mode='bicubic', align_corners=False).clamp(0, 1)
    out = torch.empty(B, T, S, S, 3)
    for t in range(T):
        oy, ox = 8 + 2 * t, 8 + t
        out[:, t] = big[:, :, oy:oy + S, ox:ox + S].permute(0, 2, 3, 1)
    return out.to(device)


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
    if loader is not None:
        clip_iter = loader.batches(start_step=start_step)
        next_hr = lambda gstep: next(clip_iter).to(dev, non_blocking=True)
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
    except KeyboardInterrupt:
        if rank == 0:
            print('main.py: KeyboardInterrupt->saving the checkpoint')
            save_checkpoint(store, FLAGS.output_dir, Net.global_step(), Net.train)
        print('main.py: quit')
        sys.exit(0)
    if rank == 0:
        save_checkpoint(store, FLAGS.output_dir, Net.global_step(), Net.train)
    print('Optimization done!!!!!!!!!!!!')
    if world > 1:
        dist.destroy_process_group()


def main(argv=None):
    FLAGS = parse_flags(argv)
    if 'LOCAL_RANK' not in os.environ:
        os.environ["CUDA_VISIBLE_DEVICES"] = FLAGS.cudaID       # reference main.py:107: overwritten unconditionally
    if FLAGS.output_dir is None:
        raise ValueError('The output directory is needed')
    os.makedirs(FLAGS.output_dir, exist_ok=True)
    if FLAGS.summary_dir:
        os.makedirs(FLAGS.summary_dir, exist_ok=True)
    if FLAGS.mode == 'inference':
        inference(FLAGS)
    elif FLAGS.mode == 'train':
        train(FLAGS)
    else:
        raise ValueError("mode must be 'inference' or 'train'")


if __name__ == '__main__':
    main()
