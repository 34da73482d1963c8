"""Generate tests/golden/*.npz by executing the REFERENCE's own Python (read from a checkout of
thunil/TecoGAN named by $TECOGAN_REFERENCE, never copied) under tests/golden/tf_shim.py:
    TECOGAN_REFERENCE=/path/to/TecoGAN python tests/golden/make_golden.py
The tests only read the committed .npz files; they never need the reference.

What the vectors pin: the reference's graph wiring (see tf_shim.py docstring).  Parameters are
regenerated at test time from the seeds stored in each file (oracle.init_*), so the fixtures
hold only inputs and outputs.
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
REF = os.environ.get("TECOGAN_REFERENCE", "TecoGAN")

from oracle import teco_oracle as O  # noqa: E402
from tests.golden import tf_shim  # noqa: E402

tf = tf_shim.install()
sys.path.insert(0, REF)
import lib.ops as ref_ops  # noqa: E402
import lib.frvsr as ref_frvsr  # noqa: E402
import lib.Teco as ref_teco  # noqa: E402
import lib.dataloader as ref_dl  # noqa: E402

ref_teco.gif_summary = lambda *a, **k: None  # observability only (SURVEY section 2 row 13)
A = tf_shim.A


class Flags(dict):
    __getattr__ = dict.__getitem__


def rnd(seed, *shape, lo=0.0, hi=1.0):
    g = torch.Generator().manual_seed(seed)
    return (torch.rand(*shape, generator=g) * (hi - lo) + lo).numpy().astype(np.float32)


def save(name, **kw):
    path = os.path.join(HERE, name + ".npz")
    np.savez_compressed(path, **kw)
    print("wrote", path, os.path.getsize(path) // 1024, "KiB")


def main():
    # ---- in-tree resamplers (lib/ops.py:126-212) and gaussDown (lib/ops.py:347-367)
    x = rnd(1, 2, 5, 7, 3)
    f = rnd(2, 2, 4, 6, 2, lo=-3, hi=3)
    hr = rnd(3, 1, 40, 44, 3)
    tf_shim.set_params({})
    save("ops", x=x, bicubic_four=np.asarray(ref_ops.bicubic_four(A(x))),
         f=f, upscale_four=np.asarray(ref_ops.upscale_four(A(f))),
         hr=hr, gauss_down=np.asarray(ref_ops.tf_data_gaussDownby4(A(hr), 1.5)),
         deprocess=np.asarray(ref_ops.deprocess(A(x))), preprocess=np.asarray(ref_ops.preprocess(A(x))))

    # ---- generator_F (lib/frvsr.py:44-88), scope 'generator' as in main.py:203 / lib/Teco.py:125
    for nrb, seed in ((3, 11), (16, 12)):
        pg = O.init_generator(seed=seed, num_resblock=nrb, bias_std=0.05)
        gi = rnd(20 + nrb, 1, 12, 10, 51)
        tf_shim.set_params(pg)
        with tf.variable_scope('generator'):
            out = ref_frvsr.generator_F(A(gi), 3, reuse=False, FLAGS=Flags(num_resblock=nrb))
        assert sorted(set(tf_shim.S.used)) == sorted(pg.keys())
        save("generator_n%d" % nrb, seed=seed, num_resblock=nrb, bias_std=0.05, inputs=gi, out=np.asarray(out))

    # ---- fnet (lib/frvsr.py:4-41), scope 'fnet' as in main.py:210 / lib/Teco.py:102
    pf = O.init_fnet(seed=31, bias_std=0.05)
    fi = rnd(32, 2, 16, 24, 6)
    tf_shim.set_params(pf)
    with tf.variable_scope('fnet'):
        out = ref_frvsr.fnet(A(fi), reuse=False)
    assert sorted(set(tf_shim.S.used)) == sorted(pf.keys())
    save("fnet", seed=31, bias_std=0.05, inputs=fi, out=np.asarray(out))

    # ---- discriminator_F (lib/Teco.py:30-74), scope 'tdiscriminator' as in lib/Teco.py:226
    pd = O.init_discriminator(seed=41, bias_std=0.05)
    di = rnd(42, 2, 32, 32, 27, lo=-1, hi=1)
    tf_shim.set_params(pd)
    with tf.variable_scope('tdiscriminator'):
        prob, layers = ref_teco.discriminator_F(A(di), FLAGS=Flags())
    assert sorted(set(tf_shim.S.used)) == sorted(pd.keys())
    save("discriminator", seed=41, bias_std=0.05, inputs=di, prob=np.asarray(prob),
         **{"layer%d" % i: np.asarray(l) for i, l in enumerate(layers)})

    # ---- VGG19_slim (lib/Teco.py:5-24)
    pv = O.init_vgg19(seed=51)
    vi = rnd(52, 1, 32, 32, 3, lo=-1, hi=1)
    tf_shim.set_params(pv)
    feats = ref_teco.VGG19_slim(A(vi), reuse=False, deep_list=O.VGG_TAPS)
    save("vgg", seed=51, inputs=vi, **{"tap%d" % i: np.asarray(feats[k]) for i, k in enumerate(O.VGG_TAPS)})

    # ---- TecoGAN()/FRVSR() forward graph + every loss scalar (lib/Teco.py:77-413)
    cases = {
        "teco_pp": dict(flags=O.TrainFlags(batch_size=1, crop_size=16, RNN_N=3, num_resblock=2), gan=True),
        "teco_nopp": dict(flags=O.TrainFlags(batch_size=2, crop_size=16, RNN_N=4, num_resblock=1, pingpang=False,
                                             vgg_scaling=-0.002), gan=True),
        "frvsr": dict(flags=O.TrainFlags.frvsr(batch_size=2, crop_size=16, RNN_N=3, num_resblock=2), gan=False),
    }
    for ci, (name, c) in enumerate(cases.items()):
        FL = c["flags"]
        P = {}
        P.update(O.init_generator(seed=61 + ci, num_resblock=FL.num_resblock, bias_std=0.05))
        P.update(O.init_fnet(seed=71 + ci, bias_std=0.05))
        P.update(O.init_discriminator(seed=81 + ci, bias_std=0.05))
        if FL.vgg_scaling > 0:
            P.update(O.init_vgg19(seed=91 + ci))
        ri = rnd(100 + ci, FL.batch_size, FL.RNN_N, FL.crop_size, FL.crop_size, 3)
        rt = rnd(200 + ci, FL.batch_size, FL.RNN_N, FL.crop_size * 4, FL.crop_size * 4, 3, lo=-1, hi=1)
        tf_shim.set_params(P)
        fl = Flags(vars(FL))
        net = ref_teco.TecoGAN(A(ri), A(rt), fl, c["gan"]) if c["gan"] else ref_teco.FRVSR(A(ri), A(rt), fl)
        save(name, ci=ci, gan=c["gan"], r_inputs=ri, r_targets=rt, gen_output=np.asarray(net.gen_output),
             update_list=np.asarray([float(v) for v in net.update_list], dtype=np.float64),
             update_list_name=np.asarray(net.update_list_name[:len(net.update_list)]),
             flags=np.asarray(repr(vars(FL))))

    # ---- calendar fixture (LR/calendar/0001..0010.png; SURVEY 8c): loader semantics lib/dataloader.py:11-50
    fl = Flags(input_dir_LR=os.path.join(REF, "LR/calendar"), input_dir_HR=None, input_dir_len=10)
    data = ref_dl.inference_data_loader(fl)
    names = [os.path.basename(p) for p in data.paths_LR]
    assert names[:6] == ["0006.png", "0005.png", "0004.png", "0003.png", "0002.png", "0001.png"], names
    frames = np.stack(data.inputs[5:])                     # 0001..0010, float32 RGB/255
    u8 = np.round(frames * 255.0).astype(np.uint8)
    assert np.array_equal(u8.astype(np.float32) / 255.0, frames)
    save("calendar_lr", full_u8=u8[:7], crop32_u8=u8[:, :32, :32], order=np.asarray(names))


if __name__ == "__main__":
    main()
