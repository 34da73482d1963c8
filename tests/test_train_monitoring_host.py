"""CPU: training monitoring of main.py --mode train --summary_dir -- the TensorBoard event writer (checked by a reader
written here, independent of tecogan_b200.summary), the validation split of the clip loader, and the logfile.txt tee."""
import glob
import hashlib
import os
import struct
import sys

import numpy as np
import pytest
import torch


class Flags:
    def __init__(self, **kw):
        self.__dict__.update(dict(input_video_dir="", input_video_pre="scene", str_dir=2000, end_dir=2001, end_dir_val=2003,
                                  max_frm=11, RNN_N=4, batch_size=2, crop_size=4, rand_seed=7, queue_thread=2,
                                  movingFirstFrame=True, random_crop=True, flip=True, mode="train"))
        self.__dict__.update(kw)


def _make_dataset(root, dirs=(2000, 2001, 2002, 2003)):
    """Random 40x52 frames; the blue channel of every pixel is 10 * (scene - 2000) + frame."""
    import cv2
    for d in dirs:
        p = os.path.join(root, "scene_%04d" % d)
        os.makedirs(p)
        rng = np.random.default_rng(d)
        for f in range(12):
            img = rng.integers(0, 256, (40, 52, 3), dtype=np.uint8)
            img[..., 2] = 10 * (d - 2000) + f
            cv2.imwrite(os.path.join(p, "col_high_%04d.png" % f), img[:, :, ::-1])


# ------------------------------------------------------------------------------------------ an independent event reader
def _crc32c(data):
    c = 0xFFFFFFFF
    for b in data:
        c ^= b
        for _ in range(8):
            c = (c >> 1) ^ (0x82F63B78 & -(c & 1))
    return c ^ 0xFFFFFFFF


def _masked(c):
    return ((((c >> 15) | (c << 17)) & 0xFFFFFFFF) + 0xA282EAD8) & 0xFFFFFFFF


def _varint(buf, pos):
    v, shift = 0, 0
    while True:
        b = buf[pos]
        pos += 1
        v |= (b & 0x7F) << shift
        if b < 0x80:
            return v, pos
        shift += 7


def _fields(buf):
    """[(field number, wire type, value)]: varints as ints, fixed64 / fixed32 as raw bytes, length-delimited as bytes."""
    out, pos = [], 0
    while pos < len(buf):
        key, pos = _varint(buf, pos)
        num, wt = key >> 3, key & 7
        if wt == 0:
            v, pos = _varint(buf, pos)
        elif wt == 1:
            v, pos = buf[pos:pos + 8], pos + 8
        elif wt == 5:
            v, pos = buf[pos:pos + 4], pos + 4
        elif wt == 2:
            n, pos = _varint(buf, pos)
            v, pos = buf[pos:pos + n], pos + n
        else:
            raise AssertionError("unexpected wire type %d" % wt)
        out.append((num, wt, v))
    return out


def read_events(path):
    """TFRecord framing with both CRCs checked, then Event / Summary / Value decoded by field number."""
    data = open(path, "rb").read()
    pos, events = 0, []
    while pos < len(data):
        header = data[pos:pos + 8]
        (n,) = struct.unpack("<Q", header)
        assert struct.unpack("<I", data[pos + 8:pos + 12])[0] == _masked(_crc32c(header))
        payload = data[pos + 12:pos + 12 + n]
        assert len(payload) == n
        assert struct.unpack("<I", data[pos + 12 + n:pos + 16 + n])[0] == _masked(_crc32c(payload))
        pos += 16 + n
        ev = {"values": []}
        for num, wt, v in _fields(payload):
            if num == 1:
                assert wt == 1
                ev["wall_time"] = struct.unpack("<d", v)[0]
            elif num == 2:
                assert wt == 0
                ev["step"] = v
            elif num == 3:
                ev["file_version"] = v.decode()
            elif num == 5:
                for vn, _, val in _fields(v):
                    assert vn == 1
                    d = {fn: fv for fn, fwt, fv in _fields(val)}
                    ev["values"].append((d[1].decode(), struct.unpack("<f", d[2])[0]))
        events.append(ev)
    return events


def _write_some(tmp_path):
    from tecogan_b200.summary import EventWriter
    w = EventWriter(str(tmp_path))
    w.add_scalars(2, [("learning_rate", 1e-4), ("l2_content_loss", 0.123456789), ("All_loss_Gen", -3.5)])
    w.add_scalars(2, [("val_l2_content_loss", 0.25)])
    w.add_scalars(300000, [("learning_rate", 5e-5)])
    w.close()
    return w.path


def test_event_file_passes_an_independent_reader(tmp_path):
    path = _write_some(tmp_path)
    name = os.path.basename(path)
    assert name.startswith("events.out.tfevents.") and name.split(".")[3].isdigit()
    ev = read_events(path)
    assert ev[0]["file_version"] == "brain.Event:2" and ev[0]["values"] == []
    assert [e["step"] for e in ev[1:]] == [2, 2, 300000]
    f32 = lambda x: float(np.float32(x))
    assert ev[1]["values"] == [("learning_rate", f32(1e-4)), ("l2_content_loss", f32(0.123456789)), ("All_loss_Gen", -3.5)]
    assert ev[2]["values"] == [("val_l2_content_loss", 0.25)]
    assert ev[3]["values"] == [("learning_rate", f32(5e-5))]
    assert all(e["wall_time"] > 1.0e9 for e in ev)


def test_event_file_reads_in_tensorboard(tmp_path):
    ea_mod = pytest.importorskip("tensorboard.backend.event_processing.event_accumulator")
    _write_some(tmp_path)
    acc = ea_mod.EventAccumulator(str(tmp_path))
    acc.Reload()
    assert sorted(acc.Tags()["scalars"]) == sorted(["learning_rate", "l2_content_loss", "All_loss_Gen", "val_l2_content_loss"])
    assert [(s.step, s.value) for s in acc.Scalars("learning_rate")] == [(2, float(np.float32(1e-4))), (300000, float(np.float32(5e-5)))]
    assert [(s.step, s.value) for s in acc.Scalars("All_loss_Gen")] == [(2, -3.5)]


def test_event_writer_flushes_every_summary(tmp_path):
    from tecogan_b200.summary import EventWriter
    w = EventWriter(str(tmp_path))
    w.add_scalars(1, [("a", 1.0)])
    assert [e.get("step") for e in read_events(w.path)][1:] == [1]      # readable before close
    w.close()


# ------------------------------------------------------------------------------------------ validation split
def _scene_of(batch):
    """Scene numbers (2000 + blue // 10) of every clip of a [B,T,h,w,3] batch."""
    blue = np.rint(batch[..., 2].numpy() * 255).astype(int)
    return set((2000 + blue // 10).reshape(-1).tolist())


def test_validation_loader_reads_only_the_held_out_scenes(tmp_path):
    from tecogan_b200.lib.dataloader import HRClipLoader, validation_loader
    root = str(tmp_path / "data")
    _make_dataset(root)
    F = Flags(input_video_dir=root)
    val, why = validation_loader(F)
    assert why is None and val.queue_thread == 1
    assert [os.path.basename(c) for c in val.clips] == ["scene_2002", "scene_2003"]
    seen = set()
    for k in range(val.steps_per_epoch * 2):
        seen |= _scene_of(val.batch(k))
    assert seen == {2002, 2003}
    train = HRClipLoader(F)
    assert [os.path.basename(c) for c in train.clips] == ["scene_2000", "scene_2001"]
    # deterministic in (rand_seed, k): a second loader, and the batch iterator, give the same batches
    val2, _ = validation_loader(F)
    it = val2.batches()
    for k in range(3):
        b = val.batch(k)
        assert torch.equal(b, val2.batch(k)) and torch.equal(b, next(it))
    other, _ = validation_loader(Flags(input_video_dir=root, rand_seed=8))
    assert not torch.equal(other.batch(0), val.batch(0))


def test_validation_draws_differ_from_training_draws(tmp_path):
    """Same scenes, same seed: a loader with the validation salt permutes and augments differently."""
    from tecogan_b200.lib.dataloader import VALIDATION_SALT, HRClipLoader
    root = str(tmp_path / "data")
    _make_dataset(root)
    F = Flags(input_video_dir=root)
    tr, va = HRClipLoader(F), HRClipLoader(F, salt=VALIDATION_SALT)
    assert tr.clips == va.clips
    assert tr._order(0).tolist() != va._order(0).tolist()
    differ = sum(not np.array_equal(tr.sample(i, 0), va.sample(i, 0)) for i in range(len(tr)))
    assert differ >= len(tr) - 2


def test_validation_skipped_without_held_out_scenes(tmp_path):
    from tecogan_b200.lib.dataloader import validation_loader
    root = str(tmp_path / "data")
    _make_dataset(root, dirs=(2000, 2001))
    val, why = validation_loader(Flags(input_video_dir=root))
    assert val is None and "No frame files" in why and "scene_2002 .. scene_2003" in why
    root2 = str(tmp_path / "data2")
    _make_dataset(root2, dirs=(2000, 2002))
    val, why = validation_loader(Flags(input_video_dir=root2, batch_size=9))      # 8 samples < one batch of 9
    assert val is None and "cannot fill one batch" in why


def test_main_prints_the_skip_line_and_keeps_training_data(tmp_path, capsys):
    import main as M
    root = str(tmp_path / "data")
    _make_dataset(root, dirs=(2000, 2001))
    assert M.validation_source(Flags(input_video_dir=root), "cpu") is None
    assert "[main] validation skipped: No frame files" in capsys.readouterr().out


def test_training_batches_unchanged(tmp_path):
    """The training loader's batches for these flags and this data set, as the loader before the validation split
    produced them (SHA-256 of the decoded float32 batches 3..12)."""
    from tecogan_b200.lib.dataloader import HRClipLoader
    root = str(tmp_path / "data")
    _make_dataset(root)
    it = HRClipLoader(Flags(input_video_dir=root)).batches(start_step=3)
    h = hashlib.sha256()
    for _ in range(10):
        h.update(next(it).numpy().tobytes())
    assert h.hexdigest() == "aa09160531828dc4ddec93c8112b9fe3ba27860a7c2abfda202dc4c06673aa3f"


def test_synthetic_validation_batches_use_their_own_seeds():
    import main as M
    F = Flags(batch_size=1, RNN_N=2, crop_size=4)
    val = M.validation_source(F, "cpu")
    v = [val(k) for k in range(3)]
    assert torch.equal(v[1], val(1)) and not torch.equal(v[0], v[1])
    for k in range(3):
        for rank in range(2):
            assert not torch.equal(v[k], M.synthetic_hr_batch(F, k, rank, "cpu"))
    assert torch.equal(M.synthetic_hr_batch(F, 5, 1, "cpu"), M.synthetic_hr_batch(F, 5, 1, "cpu", validation=False))


# ------------------------------------------------------------------------------------------ flags and logfile.txt
PARENT_FLAG_DEFAULTS = {
    'rand_seed': 1, 'input_dir_LR': None, 'input_dir_len': -1, 'input_dir_HR': None, 'mode': 'inference', 'output_dir': None,
    'output_pre': '', 'output_name': 'output', 'output_ext': 'jpg', 'summary_dir': None, 'checkpoint': None,
    'num_resblock': 16, 'pre_trained_model': False, 'vgg_ckpt': None, 'cudaID': '0', 'queue_thread': 6,
    'name_video_queue_capacity': 512, 'video_queue_capacity': 256, 'video_queue_batch': 2, 'RNN_N': 10, 'batch_size': 4,
    'flip': True, 'random_crop': True, 'movingFirstFrame': True, 'crop_size': 32, 'input_video_dir': '',
    'input_video_pre': 'scene', 'str_dir': 1000, 'end_dir': 2000, 'end_dir_val': 2050, 'max_frm': 119,
    'vgg_scaling': -0.002, 'warp_scaling': 1.0, 'pingpang': False, 'pp_scaling': 1.0, 'EPS': 1e-12, 'learning_rate': 0.0001,
    'decay_step': 500000, 'decay_rate': 0.5, 'stair': False, 'beta': 0.9, 'adameps': 1e-8, 'max_epoch': None,
    'max_iter': 1000000, 'display_freq': 20, 'summary_freq': 100, 'save_freq': 10000, 'ratio': 0.01, 'Dt_mergeDs': True,
    'Dt_ratio_0': 1.0, 'Dt_ratio_add': 0.0, 'Dt_ratio_max': 1.0, 'Dbalance': 0.4, 'crop_dt': 0.75, 'D_LAYERLOSS': True,
    'precision': 'bf16', 'train_precision': 'fp32', 'synthetic_data': False,
}


def test_flags_unchanged():
    import main as M
    assert vars(M.parse_flags([])) == PARENT_FLAG_DEFAULTS


def test_logfile_receives_stdout_and_appends(tmp_path, monkeypatch, capsys):
    import main as M
    calls = []

    def fake_inference(FLAGS):
        calls.append(FLAGS.summary_dir)
        print("frame line %d" % len(calls))
    monkeypatch.setattr(M, "inference", fake_inference)
    monkeypatch.delenv("RANK", raising=False)
    monkeypatch.setenv("CUDA_VISIBLE_DEVICES", os.environ.get("CUDA_VISIBLE_DEVICES", ""))
    out, summ = str(tmp_path / "out"), str(tmp_path / "summ")
    before = sys.stdout
    M.main(["--mode", "inference", "--output_dir", out, "--summary_dir", summ])
    assert sys.stdout is before
    M.main(["--mode", "inference", "--output_dir", out, "--summary_dir", summ])
    log = open(os.path.join(summ, "logfile.txt")).read()
    assert log == "frame line 1\nframe line 2\n"
    assert capsys.readouterr().out == log                    # still printed to the terminal
    M.main(["--mode", "inference", "--output_dir", str(tmp_path / "out2")])
    assert not glob.glob(str(tmp_path / "out2" / "*"))       # no --summary_dir: no log file anywhere
    assert open(os.path.join(summ, "logfile.txt")).read() == log
