"""CPU: the rules of the frame store's host placement -- main.frame_store_fits with host room (device, host, host loader),
the host room read from /proc/meminfo and the cgroup v2 limit, the grouping of ranks by host, and two processes sharing
one memfd mapping through an abstract Unix socket (tecogan_b200/hostmem.py)."""
import multiprocessing
import os

import numpy as np
import pytest

G = 1 << 30


def test_frame_store_fits_places_the_store_on_the_device_in_host_memory_or_nowhere():
    import main as M
    total = 80 * G                                       # device margin 4 GiB: 60 + 8 - 6 - 4 = 58 GiB of device room
    dev = (60 * G, 8 * G, 6 * G, total)
    assert M.frame_store_fits(58 * G, *dev, 100 * G)[0] == 'device'
    place, msg = M.frame_store_fits(58 * G + 1, *dev, 100 * G)
    assert place == 'host' and "does not fit in" in msg and "fits in the 100.00 GiB of host memory" in msg
    assert M.frame_store_fits(100 * G, *dev, 100 * G)[0] == 'host'              # exactly the host room
    place, msg = M.frame_store_fits(100 * G + 1, *dev, 100 * G)
    assert not place and "does not fit in the 100.00 GiB of host memory" in msg
    assert not M.frame_store_fits(1, 0, 0, 0, total, 0)[0]                     # no room anywhere
    assert M.frame_store_fits(10 * G, *dev, 0)[0] == 'device'                  # the device first, whatever the host has


def test_frame_store_fits_without_host_room_is_unchanged():
    import main as M
    dev = (60 * G, 8 * G, 6 * G, 80 * G)
    for nbytes, fits in ((10 * G, True), (58 * G, True), (58 * G + 1, False), (59 * G, False)):
        got = M.frame_store_fits(nbytes, *dev)
        assert got[0] is fits and got == M.frame_store_fits(nbytes, *dev, None)
        assert got[1] == ('frame store %.2f GiB %s the 58.00 GiB left beside a measured peak of 6.00 GiB and a 4.00 GiB '
                          'margin' % (nbytes / G, 'fits in' if fits else 'does not fit in'))


MEMINFO = "MemTotal:       %d kB\nMemFree:        1000 kB\nMemAvailable:   %d kB\nBuffers:           0 kB\n"


def _write(path, text):
    with open(str(path), "w") as f:
        f.write(text)
    return str(path)


def test_host_room_from_meminfo_and_cgroup(tmp_path):
    from tecogan_b200.hostmem import host_margin_bytes, host_room_bytes
    K = 1024
    big = _write(tmp_path / "big", MEMINFO % (1000 * G // K, 700 * G // K))       # margin 10 % of 1000 GiB = 100 GiB
    small = _write(tmp_path / "small", MEMINFO % (16 * G // K, 10 * G // K))     # margin 4 GiB
    nocg = str(tmp_path / "no_cgroup")
    os.makedirs(nocg)
    assert host_margin_bytes(1000 * G) == 100 * G and host_margin_bytes(16 * G) == 4 * G
    assert host_room_bytes(big, nocg) == 600 * G
    assert host_room_bytes(small, nocg) == 6 * G
    assert host_room_bytes(_write(tmp_path / "tiny", MEMINFO % (8 * G // K, 3 * G // K)), nocg) == 0
    unlimited = str(tmp_path / "unlimited")
    os.makedirs(unlimited)
    _write(os.path.join(unlimited, "memory.max"), "max\n")
    _write(os.path.join(unlimited, "memory.current"), "%d\n" % (50 * G))
    assert host_room_bytes(big, unlimited) == 600 * G
    limited = str(tmp_path / "limited")
    os.makedirs(limited)
    _write(os.path.join(limited, "memory.max"), "%d\n" % (300 * G))
    _write(os.path.join(limited, "memory.current"), "%d\n" % (40 * G))
    assert host_room_bytes(big, limited) == 160 * G                          # min(700, 300 - 40) - 100
    _write(os.path.join(limited, "memory.max"), "%d\n" % (900 * G))
    assert host_room_bytes(big, limited) == 600 * G                          # the limit is above MemAvailable


def test_cgroup_dir_follows_proc_self_cgroup(tmp_path):
    from tecogan_b200.hostmem import cgroup_dir
    root = str(tmp_path / "cg")
    os.makedirs(os.path.join(root, "user.slice", "job"))
    assert cgroup_dir(_write(tmp_path / "c1", "0::/user.slice/job\n"), root) == os.path.join(root, "user.slice", "job")
    assert cgroup_dir(_write(tmp_path / "c2", "0::/\n"), root) == os.path.join(root, "")
    assert cgroup_dir(_write(tmp_path / "c3", "0::/not/visible\n"), root) == root
    assert cgroup_dir(str(tmp_path / "missing"), root) == root


def test_node_groups():
    from tecogan_b200.hostmem import node_groups
    assert node_groups(["a"]) == [(0,)]
    assert node_groups(["a", "b", "a", "c", "b"]) == [(0, 2), (1, 4), (0, 2), (3,), (1, 4)]
    assert node_groups(["n1"] * 4 + ["n2"] * 4) == [(0, 1, 2, 3)] * 4 + [(4, 5, 6, 7)] * 4


def _peer(name, nbytes, conn):
    from tecogan_b200.hostmem import HostMapping, receive_fd
    m = HostMapping.from_fd(receive_fd(name), nbytes)
    a = m.array()
    conn.send((m.inode, int(a[:nbytes // 2].sum()), [l for l in open("/proc/self/maps") if "tecogan-frame-store" in l]))
    a[nbytes // 2:] = 7                         # the second half, for the creator to see
    del a
    m.close()
    conn.send("done")


def test_two_processes_share_one_memfd_mapping():
    from tecogan_b200.hostmem import HostMapping, fd_server, send_fd
    shm = sorted(os.listdir("/dev/shm")) if os.path.isdir("/dev/shm") else []
    nbytes = 3 * 4096 + 5
    m = HostMapping.create(nbytes)
    a = m.array()
    assert a.shape == (nbytes,) and m.size == 4 * 4096
    a[:nbytes // 2] = np.arange(nbytes // 2) % 251
    sock, name = fd_server(1)
    ctx = multiprocessing.get_context("spawn")
    parent, child = ctx.Pipe()
    p = ctx.Process(target=_peer, args=(name, nbytes, child))
    p.start()
    try:
        send_fd(sock, m.fd, 1)
        inode, total, maps = parent.recv()
        assert parent.recv() == "done"
    finally:
        p.join(60)
        sock.close()
    assert p.exitcode == 0
    assert inode == m.inode and total == int((np.arange(nbytes // 2) % 251).sum())
    assert maps and all("/memfd:tecogan-frame-store" in l for l in maps)
    assert (a[nbytes // 2:] == 7).all()
    assert name.startswith("\0") and not os.path.exists(name[1:])
    assert (sorted(os.listdir("/dev/shm")) if os.path.isdir("/dev/shm") else []) == shm
    del a
    m.close()
    m.close()                                   # releasing twice is a no-op
    assert not [l for l in open("/proc/self/maps") if "tecogan-frame-store" in l]


def test_a_mapping_nothing_refers_to_is_unmapped():
    import gc
    from tecogan_b200.hostmem import HostMapping
    m = HostMapping.create(100)
    m.close_fd()
    a = m.array()
    del m
    gc.collect()
    a[:] = 1                                    # the array keeps the mapping alive
    assert [l for l in open("/proc/self/maps") if "tecogan-frame-store" in l]
    del a
    gc.collect()
    assert not [l for l in open("/proc/self/maps") if "tecogan-frame-store" in l]


def _setup_worker(rank, world, init, fail, out_dir):
    """One gloo rank calling shared_mapping with a failure injected on one rank: `fail` is (rank, 'create' | 'register')."""
    import torch.distributed as dist
    from tecogan_b200 import hostmem
    who, what = fail

    def broken(*a, **k):
        raise (OSError(28, "no space left (injected)") if what == "create" else RuntimeError("register refused (injected)"))
    if what == "create" and rank == who:
        hostmem.HostMapping.create = classmethod(lambda cls, n: broken())
    if what == "register":                      # no device here: every rank but `who` registers as a no-op
        hostmem.HostMapping.register = lambda self: broken() if rank == who else 0
    dist.init_process_group("gloo", init_method=init, rank=rank, world_size=world)
    try:
        try:
            m, node = hostmem.shared_mapping(5000, rank, world)
            res = "ok %d %s" % (m.inode, node)
            m.close()
        except hostmem.HostStoreError as e:
            res = "error " + str(e)
        with open(os.path.join(out_dir, "rank%d" % rank), "w") as f:
            f.write(res + "\n" + "".join(l for l in open("/proc/self/maps") if "tecogan-frame-store" in l))
    finally:
        dist.destroy_process_group()


def _run_setup(tmp_path, fail):
    import torch.multiprocessing as mp
    mp.spawn(_setup_worker, args=(3, "file://" + str(tmp_path / "rendezvous"), fail, str(tmp_path)), nprocs=3, join=True)
    return [open(str(tmp_path / ("rank%d" % r))).read().split("\n", 1) for r in range(3)]


def test_shared_mapping_is_one_memfd_for_the_ranks_of_a_host(tmp_path):
    got = _run_setup(tmp_path, (-1, "register"))
    assert all(res.startswith("ok ") for res, _ in got), got
    assert len({res for res, _ in got}) == 1 and got[0][0].endswith("(0, 1, 2)")     # one inode, one node
    assert all(not maps.strip() for _, maps in got)                                 # every rank released it


@pytest.mark.parametrize("fail", [(0, "create"), (0, "register"), (2, "register")])
def test_a_failure_on_one_rank_reaches_every_rank(tmp_path, fail):
    """A rank that cannot create or register the host store does not leave the others waiting: every rank raises
    HostStoreError naming the failed rank, and no rank keeps a mapping."""
    got = _run_setup(tmp_path, fail)
    for res, maps in got:
        assert res.startswith("error the host frame store could not be set up: rank %d: " % fail[0]), res
        assert "injected" in res and not maps.strip()
