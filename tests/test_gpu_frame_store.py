"""GPU: the device frame store (tecogan_b200/lib/dataloader.py::FrameStore, teco_gather_clips_u8) serves the host
loader's batches bit for bit -- over epochs, with and without moving-first-frame and flip, on each rank's shard, for the
validation loader's salted draws and from a resumed step -- and so do the LR inputs and targets frvsr_gpu_data_loader
makes of them; several ranks build byte-identical stores; main.py --mode train --input_video_dir selects the store and
feeds training and validation the batches the host loader would have."""
import os

import numpy as np
import pytest
import torch

from tests.test_dataloader_host import Flags
from tests.test_frame_store_host import _scenes

pytestmark = pytest.mark.gpu

SIZES = [(40, 52), (36, 36), (47, 61), (64, 40)]     # 36 x 36: the 24-pixel crop after the largest moving-first-frame shrink


def _same(a, b):
    return a.shape == b.shape and a.dtype == b.dtype and torch.equal(a.view(torch.int32), b.view(torch.int32))


@pytest.fixture(scope="module")
def data(tmp_path_factory):
    root = str(tmp_path_factory.mktemp("frames"))
    _scenes(root, SIZES + [(44, 50), (38, 45)], frames=10, seed=7)      # 2004, 2005: held-out scenes
    return root


def _flags(root, **kw):
    return Flags(**dict(dict(input_video_dir=root, str_dir=2000, end_dir=2003, end_dir_val=2005, max_frm=9, RNN_N=4,
                             batch_size=3, crop_size=4), **kw))


@pytest.mark.parametrize("moving,flip", [(True, True), (False, True), (True, False), (False, False)])
@pytest.mark.parametrize("rank,world", [(0, 1), (0, 2), (1, 2)])
def test_store_batches_equal_the_host_loader(data, moving, flip, rank, world):
    from tecogan_b200.lib.dataloader import FrameStore, HRClipLoader, frvsr_gpu_data_loader
    F = _flags(data, movingFirstFrame=moving, flip=flip)
    L = HRClipLoader(F, rank=rank, world=world)
    store = FrameStore([L], "cuda")
    assert store.nbytes == FrameStore.estimate_bytes([L]) == 10 * 3 * sum(h * w for h, w in SIZES)
    steps = range(0, 2 * L.steps_per_epoch + 2)                          # into a third epoch
    for k in steps:
        host = L.batch(k).cuda()
        dev = store.batch(k)
        assert _same(dev, host), k
        for a, b in zip(frvsr_gpu_data_loader(dev, F), frvsr_gpu_data_loader(host, F)):
            assert _same(a, b), k
    it = store.batches(start_step=5)                                     # a resumed run
    for k in range(5, 5 + L.steps_per_epoch + 1):
        assert _same(next(it), L.batch(k).cuda()), k


def test_validation_view_equals_the_validation_loader(data):
    from tecogan_b200.lib.dataloader import FrameStore, HRClipLoader, validation_loader
    F = _flags(data)
    L = HRClipLoader(F)
    V, why = validation_loader(F)
    assert V is not None, why
    store = FrameStore([L, V], "cuda")
    assert store.nbytes == 10 * 3 * sum(h * w for h, w in SIZES + [(44, 50), (38, 45)])
    vs = store.view(V)
    for k in range(2 * V.steps_per_epoch + 1):
        assert _same(vs.batch(k), V.batch(k).cuda()), k
        assert _same(store.batch(k), L.batch(k).cuda()), k
    with pytest.raises(ValueError, match="not built from this loader"):
        store.view(HRClipLoader(F))


def test_gather_kernel_checks_its_arguments():
    from tecogan_b200 import kernels as K
    buf = torch.zeros(64, dtype=torch.uint8, device="cuda")
    with pytest.raises(ValueError, match="teco_gather_clips_u8"):
        K.gather_clips_u8(buf, torch.zeros((0, 3), dtype=torch.int64, device="cuda"), 2)
    t = torch.tensor([[0, 6, 0], [0, 6, 1]], dtype=torch.int64, device="cuda")
    buf = torch.arange(64, dtype=torch.uint8, device="cuda")
    out = K.gather_clips_u8(buf, t, 2).cpu().numpy()
    ref = np.arange(12, dtype=np.float32).reshape(2, 2, 3) / np.float32(255.0)
    assert np.array_equal(out[0], ref) and np.array_equal(out[1], ref[:, ::-1])


def _rank_worker(rank, world, backend, init, root, out_dir):
    import torch.distributed as dist
    from tecogan_b200.lib.dataloader import FrameStore, HRClipLoader, validation_loader
    dev = torch.device("cuda", rank if backend == "nccl" else 0)
    torch.cuda.set_device(dev)
    kw = dict(device_id=dev) if backend == "nccl" else {}
    dist.init_process_group(backend, init_method=init, rank=rank, world_size=world, **kw)
    try:
        F = _flags(root)
        L = HRClipLoader(F, rank=rank, world=world)
        store = FrameStore([L, validation_loader(F)[0]], dev, rank=rank, world=world, chunk_bytes=20000)
        with open(os.path.join(out_dir, "rank%d" % rank), "w") as f:
            f.write(store.checksum())
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize("backend", ["gloo", "nccl"])
def test_ranks_build_identical_stores(data, tmp_path, backend):
    """Each rank decodes its share and broadcasts it; every rank ends with the single-process store.  gloo runs both ranks
    on one device; NCCL needs a device per rank."""
    import torch.multiprocessing as mp
    from tecogan_b200.lib.dataloader import FrameStore, HRClipLoader, validation_loader
    if backend == "nccl" and torch.cuda.device_count() < 2:
        pytest.skip("NCCL ranks need two devices")
    F = _flags(data)
    ref = FrameStore([HRClipLoader(F), validation_loader(F)[0]], "cuda").checksum()
    mp.spawn(_rank_worker, args=(2, backend, "file://" + str(tmp_path / "rendezvous"), data, str(tmp_path)), nprocs=2)
    for r in range(2):
        assert open(str(tmp_path / ("rank%d" % r))).read() == ref, r


def test_main_train_from_disk_selects_the_store_and_feeds_the_host_batches(tmp_path, monkeypatch, capsys):
    """Two short runs of main.train on the same scenes, one on the store and one held to the host loader: the HR batches
    handed to frvsr_gpu_data_loader -- every training step's and every validation pass's, in order -- are identical."""
    import main as M
    import tecogan_b200.lib.dataloader as D
    from tecogan_b200 import config
    data = str(tmp_path / "frames")
    # crop 16 (FNet pools 16x16 LR frames three times): 72-pixel windows; 80 x 80 is that after the largest 3-frame shrink
    _scenes(data, [(84, 96), (80, 80), (90, 101), (96, 84), (82, 88), (88, 90)], frames=10, seed=3)
    original = D.frvsr_gpu_data_loader

    def run(name, force_host):
        seen = []

        def recording(hr, FLAGS):
            seen.append(hr.detach().cpu().clone())
            return original(hr, FLAGS)
        monkeypatch.setattr(D, "frvsr_gpu_data_loader", recording)
        if force_host:
            monkeypatch.setattr(M, "frame_store_fits", lambda *a: (False, "held to the host loader"))
        F = M.parse_flags(["--mode", "train", "--input_video_dir", data, "--str_dir", "2000", "--end_dir", "2003",
                           "--end_dir_val", "2005", "--max_frm", "9", "--RNN_N", "3", "--batch_size", "2", "--crop_size", "16",
                           "--num_resblock", "2", "--ratio", "-0.01", "--max_iter", "7", "--summary_freq", "3",
                           "--save_freq", "100", "--display_freq", "100", "--queue_thread", "2", "--precision", "fp32",
                           "--output_dir", str(tmp_path / name), "--summary_dir", str(tmp_path / (name + "_summ"))])
        os.makedirs(F.output_dir)
        monkeypatch.chdir(str(tmp_path))
        prev = config.precision(), config.train_precision()
        try:
            M.train(F)
        finally:
            config.set_precision(prev[0])
            config.set_train_precision(prev[1])
            monkeypatch.undo()
        return seen, capsys.readouterr().out

    store_seen, store_out = run("store", False)
    host_seen, host_out = run("host", True)
    assert "training reads its clips from the frame store on the device" in store_out
    assert "[main] frame store: 60 frames" in store_out
    assert "training reads its clips from the host loader" in host_out
    assert store_out.count("-----------Validation data scalars-----------") == 2       # steps 3 and 6
    assert len(store_seen) == len(host_seen) == 1 + 7 + 2          # the shape-only batch, 7 steps, 2 validation passes
    for i, (a, b) in enumerate(zip(store_seen, host_seen)):
        assert _same(a, b), i
