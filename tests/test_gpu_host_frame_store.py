"""GPU: the frame store's host placement (tecogan_b200/lib/dataloader.py::FrameStore(placement='host'),
teco_gather_clips_host_u8) serves the host loader's and the device store's batches bit for bit -- over epochs, with and
without moving-first-frame and flip, on each rank's shard, from a resumed step, through the validation view and through
frvsr_gpu_data_loader; the kernel matches numpy at every source alignment; batches handed out stay intact while the
iterator prefetches; a failed registration leaves no CUDA error behind; two ranks on one host share one memfd store;
main.py --mode train --input_video_dir places the store in host memory when the device has no room and feeds training
the host loader's batches, and trains through the host loader when the registration fails."""
import ctypes
import os

import numpy as np
import pytest
import torch

from tests.test_frame_store_host import _scenes
from tests.test_gpu_frame_store import SIZES, _flags, _same, data  # noqa: F401  (data: the module's scenes fixture)

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("moving,flip", [(True, True), (False, True), (True, False), (False, False)])
@pytest.mark.parametrize("rank,world", [(0, 1), (0, 2), (1, 2)])
def test_host_store_batches_equal_the_host_loader_and_the_device_store(data, moving, flip, rank, world):  # noqa: F811
    from tecogan_b200.lib.dataloader import FrameStore, HRClipLoader, frvsr_gpu_data_loader
    F = _flags(data, movingFirstFrame=moving, flip=flip)
    L = HRClipLoader(F, rank=rank, world=world)
    store = FrameStore([L], "cuda", placement="host", chunk_bytes=30000)
    dstore = FrameStore([L], "cuda")
    try:
        assert store.placement == "host" and not store.buf.is_cuda
        assert store.nbytes == dstore.nbytes == 10 * 3 * sum(h * w for h, w in SIZES)
        assert store.checksum() == dstore.checksum()
        for k in range(0, 2 * L.steps_per_epoch + 2):                    # into a third epoch
            host = L.batch(k).cuda()
            got = store.batch(k)
            assert _same(got, host) and _same(got, dstore.batch(k)), k
            for a, b in zip(frvsr_gpu_data_loader(got, F), frvsr_gpu_data_loader(host, F)):
                assert _same(a, b), k
        it = store.batches(start_step=5)                                 # a resumed run
        for k in range(5, 5 + L.steps_per_epoch + 1):
            assert _same(next(it), L.batch(k).cuda()), k
        it.close()
    finally:
        store.close()


def test_host_store_validation_view_equals_the_validation_loader(data):  # noqa: F811
    from tecogan_b200.lib.dataloader import FrameStore, HRClipLoader, validation_loader
    F = _flags(data)
    L = HRClipLoader(F)
    V, why = validation_loader(F)
    assert V is not None, why
    store = FrameStore([L, V], "cuda", placement="host")
    try:
        vs = store.view(V)
        for k in range(2 * V.steps_per_epoch + 1):
            assert _same(vs.batch(k), V.batch(k).cuda()), k
            assert _same(store.batch(k), L.batch(k).cuda()), k
    finally:
        store.close()


def test_prefetched_batches_are_waited_for_and_not_reused_while_read(data):  # noqa: F811
    """The iterator gathers batch k + 1 on its own stream as soon as it hands out batch k.  Each batch is compared on the
    caller's stream right after next(), with no synchronisation: only the wait on the gather's event orders the two.
    Batches the caller holds stay intact; a batch the caller drops while its stream still has to read it (behind a
    sleep) is not handed to the next gather (record_stream)."""
    from tecogan_b200.lib.dataloader import FrameStore, HRClipLoader
    F = _flags(data)
    L = HRClipLoader(F)
    store = FrameStore([L], "cuda", placement="host")
    try:
        refs = [L.batch(3 + i).cuda() for i in range(16)]
        torch.cuda.synchronize()
        it = store.batches(start_step=3)
        held, copies = [], []
        for i in range(16):
            b = next(it)
            assert _same(b, refs[i]), i
            if i < 6:
                held.append(b)
                continue
            torch.cuda._sleep(50_000_000)       # the caller's stream is busy for a while before it reads b
            copies.append((i, b.clone()))
            del b                               # dropped while that read is still queued
        torch.cuda.synchronize()
        for i, b in enumerate(held):
            assert _same(b, refs[i]), i
        for i, c in copies:
            assert _same(c, refs[i]), i
        it.close()
    finally:
        store.close()


def _mapped(nbytes, seed):
    from tecogan_b200.hostmem import HostMapping
    m = HostMapping.create(nbytes)
    m.close_fd()
    a = m.array()
    a[:] = np.random.default_rng(seed).integers(0, 256, nbytes, dtype=np.uint8)
    m.register()
    return m, a


@pytest.mark.parametrize("S", [1, 2, 5, 24, 136, 200])
def test_host_gather_kernel_matches_numpy_at_every_alignment(S):
    """Source rows start at every residue mod 16 (an odd frame width makes the pitch odd, so the rows of one window
    start at every residue too), flipped and not, and one window ends at the store's last byte; the output also equals
    teco_gather_clips_u8 on a device copy of the store."""
    from tecogan_b200 import kernels as K
    W = S + 17 if S % 2 == 0 else S + 16          # odd width
    pitch = 3 * W
    nbytes = (S + 3) * pitch + 64
    m, a = _mapped(nbytes, S)
    try:
        rows = [(r + 16 * ((r * 7 + f) % 3), pitch, f) for r in range(16) for f in (0, 1)]
        rows += [(nbytes - (S - 1) * pitch - 3 * S, pitch, f) for f in (0, 1)]
        assert all(off + (S - 1) * p + 3 * S <= nbytes for off, p, _ in rows)
        assert {off % 16 for off, _, _ in rows} == set(range(16))
        t = torch.from_numpy(np.array(rows, np.int64)).cuda()
        got = K.gather_clips_host_u8(m.dev_addr, t, S).cpu().numpy()
        for i, (off, p, f) in enumerate(rows):
            win = np.stack([a[off + y * p:off + y * p + 3 * S].reshape(S, 3) for y in range(S)])
            if f:
                win = win[:, ::-1]
            ref = np.divide(win.astype(np.float32), np.float32(255.0))
            assert np.array_equal(got[i].view(np.uint32), ref.view(np.uint32)), (i, off % 16, f)
        dev = torch.from_numpy(a.copy()).cuda()
        assert np.array_equal(got.view(np.uint32), K.gather_clips_u8(dev, t, S).cpu().numpy().view(np.uint32))
    finally:
        del a
        m.close()


def test_host_gather_kernel_checks_its_arguments():
    from tecogan_b200 import _ffi, kernels as K
    m, a = _mapped(4096, 0)
    try:
        one = torch.zeros((1, 3), dtype=torch.int64, device="cuda")
        out = torch.empty(64, device="cuda")
        s = _ffi.stream_ptr()
        for args in ((0, one.data_ptr(), 1, 2, out.data_ptr()),            # NULL store
                     (m.dev_addr, 0, 1, 2, out.data_ptr()),                # NULL table
                     (m.dev_addr, one.data_ptr(), 1, 2, 0),                # NULL out
                     (m.dev_addr, one.data_ptr(), 0, 2, out.data_ptr()),   # n = 0
                     (m.dev_addr, one.data_ptr(), 65536, 2, out.data_ptr()),
                     (m.dev_addr, one.data_ptr(), 1, 0, out.data_ptr()),   # S <= 0
                     (m.dev_addr, one.data_ptr(), 1, -3, out.data_ptr())):
            with pytest.raises(ValueError, match="teco_gather_clips_host_u8"):
                _ffi.call("teco_gather_clips_host_u8", args[0], ctypes.c_void_p(args[1]), args[2], args[3],
                          ctypes.c_void_p(args[4]), s)
        with pytest.raises(ValueError, match="teco_gather_clips_host_u8"):
            K.gather_clips_host_u8(m.dev_addr, torch.zeros((65536, 3), dtype=torch.int64, device="cuda"), 1)
        with pytest.raises(ValueError, match="teco_host_register"):
            _ffi.call("teco_host_register", ctypes.c_void_p(0), ctypes.c_size_t(4096), ctypes.byref(ctypes.c_void_p()))
        with pytest.raises(RuntimeError, match="teco_host_register: cudaHostRegister failed"):
            m.register()                        # the range is registered already
        t = torch.tensor([[0, 6, 1]], dtype=torch.int64, device="cuda")
        got = K.gather_clips_host_u8(m.dev_addr, t, 2)      # the failure left no error for this launch to report
        ref = np.divide(a[:12].reshape(2, 2, 3)[:, ::-1].astype(np.float32), np.float32(255.0))
        assert np.array_equal(got[0].cpu().numpy(), ref)
        with pytest.raises(ValueError, match="teco_host_unregister"):
            _ffi.call("teco_host_unregister", ctypes.c_void_p(0))
    finally:
        del a
        m.close()


def _rank_worker(rank, world, init, root, out_dir):
    import torch.distributed as dist
    from tecogan_b200.lib.dataloader import FrameStore, HRClipLoader, validation_loader
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    dist.init_process_group("gloo", init_method=init, rank=rank, world_size=world)
    try:
        F = _flags(root)
        L = HRClipLoader(F, rank=rank, world=world)
        store = FrameStore([L, validation_loader(F)[0]], dev, rank=rank, world=world, chunk_bytes=20000, placement="host")
        same = all(_same(store.batch(k), L.batch(k).cuda()) for k in range(L.steps_per_epoch + 1))
        with open(os.path.join(out_dir, "rank%d" % rank), "w") as f:
            f.write("%s %d %d" % (store.checksum(), store._host.inode, int(same)))
        dist.barrier()                      # neither rank releases the store before both have read it
        store.close()
    finally:
        dist.destroy_process_group()


def test_two_ranks_share_one_host_store(data, tmp_path):  # noqa: F811
    """Two gloo ranks on one device: rank 0 creates the memfd store, rank 1 receives it over the abstract socket, each
    decodes half of the frames; both see the single-process store and cut the host loader's batches of their shard."""
    import torch.multiprocessing as mp
    from tecogan_b200.lib.dataloader import FrameStore, HRClipLoader, validation_loader
    F = _flags(data)
    ref = FrameStore([HRClipLoader(F), validation_loader(F)[0]], "cuda").checksum()
    mp.spawn(_rank_worker, args=(2, "file://" + str(tmp_path / "rendezvous"), data, str(tmp_path)), nprocs=2, join=True)
    got = [open(str(tmp_path / ("rank%d" % r))).read().split() for r in range(2)]
    assert got[0][0] == got[1][0] == ref
    assert got[0][1] == got[1][1]                   # one memfd: the same inode on both ranks
    assert got[0][2] == got[1][2] == "1"


def test_main_train_from_disk_places_the_store_in_host_memory(tmp_path, monkeypatch, capsys):
    """main.train with no device room for the store and host room for it: the store goes to host memory, and the HR
    batches handed to frvsr_gpu_data_loader -- every training step's and every validation pass's, in order -- are those
    of a run held to the host loader."""
    import main as M
    import tecogan_b200.lib.dataloader as D
    from tecogan_b200 import config
    data = str(tmp_path / "frames")
    _scenes(data, [(84, 96), (80, 80), (90, 101), (96, 84), (82, 88), (88, 90)], frames=10, seed=3)
    original, fits = D.frvsr_gpu_data_loader, M.frame_store_fits

    def run(name, host_room):
        seen = []

        def recording(hr, FLAGS):
            seen.append(hr.detach().cpu().clone())
            return original(hr, FLAGS)
        monkeypatch.setattr(D, "frvsr_gpu_data_loader", recording)
        monkeypatch.setattr(M, "node_host_room", lambda rank, world: host_room)
        monkeypatch.setattr(M, "frame_store_fits", lambda s, free, reserved, peak, total, host=None:
                            fits(s, 0, 0, peak, total, host))                 # no device room
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

    store_seen, store_out = run("hoststore", 1 << 30)
    host_seen, host_out = run("loader", 0)
    from tecogan_b200.hostmem import HostMapping
    register = HostMapping.register

    def twice(self):                            # a registration that fails in CUDA: the range is registered already
        register(self)
        return register(self)
    monkeypatch.setattr(HostMapping, "register", twice)
    fail_seen, fail_out = run("regfail", 1 << 30)
    assert "training reads its clips from the frame store in host memory" in store_out
    assert "[main] frame store: 60 frames" in store_out
    assert "training reads its clips from the host loader" in host_out
    assert "the host frame store could not be set up" in fail_out and "cudaHostRegister failed" in fail_out
    assert "training reads its clips from the host loader" in fail_out and "[main] frame store:" not in fail_out
    for out in (store_out, host_out, fail_out):
        assert out.count("-----------Validation data scalars-----------") == 2
    assert len(store_seen) == len(host_seen) == len(fail_seen) == 1 + 7 + 2
    for i, (a, b, c) in enumerate(zip(store_seen, host_seen, fail_seen)):
        assert _same(a, b) and _same(c, b), i
