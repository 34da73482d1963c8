"""Host memory for the frame store's host placement (lib/dataloader.py::FrameStore): one anonymous memfd mapping per node,
shared by that node's ranks, page-locked and mapped into the device's address space.

The lowest rank on a host creates the memfd (os.memfd_create + ftruncate) and maps it MAP_SHARED; the other ranks on that
host receive its file descriptor over an abstract-namespace Unix socket (SCM_RIGHTS) and map it too.  Nothing is created
in a file system, so nothing outlives the processes, and a small /dev/shm does not limit the size.  How much of the
host's memory the store may take is host_room_bytes()."""
import ctypes
import mmap
import os
import secrets
import socket
import weakref

import numpy as np

GiB = 1 << 30
PAGE = mmap.PAGESIZE

_libc = ctypes.CDLL(None, use_errno=True)
_libc.mmap.restype = ctypes.c_void_p
_libc.mmap.argtypes = [ctypes.c_void_p, ctypes.c_size_t, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_long]
_libc.munmap.restype = ctypes.c_int
_libc.munmap.argtypes = [ctypes.c_void_p, ctypes.c_size_t]
_MAP_FAILED = ctypes.c_void_p(-1).value


SHARE_TIMEOUT_S = 300          # a peer that has not connected (or a lead that has not sent) by then has failed


class HostStoreError(RuntimeError):
    """The host store's memory could not be created, shared or registered with the device on some rank."""


def host_margin_bytes(total_bytes):
    """Host memory kept free beside a host-placed store: max(4 GiB, 10 % of MemTotal) -- the pinned batch and table
    buffers, the Python heap, the loaders' decode threads and the rest of the node."""
    return max(4 * GiB, total_bytes // 10)


def _meminfo(text):
    out = {}
    for line in text.splitlines():
        key, _, rest = line.partition(':')
        parts = rest.split()
        if parts:
            out[key.strip()] = int(parts[0]) * (1024 if parts[1:] == ['kB'] else 1)
    return out


def _read(path):
    try:
        with open(path) as f:
            return f.read()
    except OSError:
        return None


def cgroup_dir(proc_cgroup='/proc/self/cgroup', root='/sys/fs/cgroup'):
    """This process's cgroup v2 directory (the '0::<path>' line of /proc/self/cgroup under `root`), or `root` when that
    directory is not visible (a cgroup namespace shows its own cgroup as the root)."""
    for line in (_read(proc_cgroup) or '').splitlines():
        if line.startswith('0::'):
            d = os.path.join(root, line[3:].strip().lstrip('/'))
            if os.path.isdir(d):
                return d
    return root


def host_room_bytes(meminfo='/proc/meminfo', cgroup=None):
    """Bytes of host memory a host-placed frame store may take: MemAvailable, capped by the cgroup v2 limit
    memory.max - memory.current of `cgroup` (cgroup_dir() by default) when one is set, minus host_margin_bytes(MemTotal).
    Only reads; never below 0."""
    info = _meminfo(_read(meminfo) or '')
    avail, total = info.get('MemAvailable', 0), info.get('MemTotal', 0)
    cg = cgroup_dir() if cgroup is None else cgroup
    lim, cur = (_read(os.path.join(cg, name)) for name in ('memory.max', 'memory.current'))
    if lim is not None and cur is not None and lim.strip() != 'max':
        avail = min(avail, int(lim) - int(cur))
    return max(0, avail - host_margin_bytes(total))


def node_groups(hostnames):
    """hostnames[r] is rank r's host name -> for each rank, the sorted tuple of ranks on its host (the first of which
    creates that host's mapping)."""
    by_host = {}
    for r, h in enumerate(hostnames):
        by_host.setdefault(h, []).append(r)
    return [tuple(by_host[h]) for h in hostnames]


def fd_server(peers):
    """A listening abstract-namespace Unix socket for `peers` connections -> (socket, name).  The name is random and
    lives in no file system."""
    sock = socket.socket(socket.AF_UNIX, socket.SOCK_STREAM)
    name = '\0tecogan-frame-store-%d-%s' % (os.getpid(), secrets.token_hex(8))
    sock.bind(name)
    sock.listen(max(1, peers))
    return sock, name


def send_fd(sock, fd, peers):
    """Hands `fd` to `peers` connections on `sock` (SCM_RIGHTS); a connection from another user is dropped."""
    sent = 0
    while sent < peers:
        conn, _ = sock.accept()
        with conn:
            pid, uid, gid = np.frombuffer(conn.getsockopt(socket.SOL_SOCKET, socket.SO_PEERCRED, 12), np.int32)
            if int(uid) != os.getuid():
                continue
            socket.send_fds(conn, [b'F'], [fd])
            sent += 1


def receive_fd(name, timeout=SHARE_TIMEOUT_S):
    """The file descriptor the fd_server called `name` hands out."""
    with socket.socket(socket.AF_UNIX, socket.SOCK_STREAM) as sock:
        sock.settimeout(timeout)
        sock.connect(name)
        _, fds, _, _ = socket.recv_fds(sock, 1, 1)
    if len(fds) != 1:
        raise RuntimeError('receive_fd: no file descriptor from %r' % name)
    return fds[0]


def _release(state):
    """Waits for the device the mapping was registered on (a prefetched gather may still read it), unregisters, then
    unmaps; raises what any of them reports.  Runs once."""
    addr, size, device = state.pop('addr', None), state['size'], state.pop('device', None)
    if addr is None:
        return
    if device is not None:
        import torch
        from . import _ffi
        torch.cuda.synchronize(device)
        _ffi.call('teco_host_unregister', ctypes.c_void_p(addr))
    if _libc.munmap(ctypes.c_void_p(addr), size) != 0:
        e = ctypes.get_errno()
        raise OSError(e, 'munmap of the frame store mapping failed: ' + os.strerror(e))


class _View:
    """numpy's handle on the mapping; holds the HostMapping so the memory stays mapped while an array uses it."""

    def __init__(self, owner, nbytes):
        self.owner = owner
        self.__array_interface__ = {'shape': (nbytes,), 'typestr': '|u1', 'data': (owner.addr, False), 'version': 3}


class HostMapping:
    """`nbytes` of a memfd mapped MAP_SHARED (the size rounded up to whole pages, so 16-byte-aligned reads past the last
    byte stay inside it).  create() makes a new memfd; from_fd() maps one received from another process.  register()
    page-locks it and maps it into the current device's address space (teco_host_register) -> device address.  close()
    waits for that device, unregisters, then unmaps, and raises their errors; a mapping nothing refers to any more is
    released the same way (from the garbage collector, where errors can only be printed)."""

    def __init__(self, fd, nbytes):
        self.nbytes = int(nbytes)
        self.size = max(PAGE, -(-self.nbytes // PAGE) * PAGE)
        self.inode = os.fstat(fd).st_ino
        addr = _libc.mmap(None, self.size, mmap.PROT_READ | mmap.PROT_WRITE, mmap.MAP_SHARED, fd, 0)
        if addr in (None, _MAP_FAILED):
            e = ctypes.get_errno()
            raise OSError(e, 'mmap of %d bytes for the frame store failed: %s' % (self.size, os.strerror(e)))
        self.addr, self.dev_addr = addr, None
        self._state = {'addr': addr, 'size': self.size}
        self._finalizer = weakref.finalize(self, _release, self._state)
        self._finalizer.atexit = False            # process exit releases both

    @classmethod
    def create(cls, nbytes):
        fd = os.memfd_create('tecogan-frame-store', os.MFD_CLOEXEC)
        try:
            os.ftruncate(fd, max(PAGE, -(-int(nbytes) // PAGE) * PAGE))
            m = cls(fd, nbytes)
            m.fd = fd                               # kept open until handed out (send_fd), then close_fd()
            return m
        except BaseException:
            os.close(fd)
            raise

    @classmethod
    def from_fd(cls, fd, nbytes):
        try:
            return cls(fd, nbytes)
        finally:
            os.close(fd)

    def close_fd(self):
        fd, self.fd = getattr(self, 'fd', None), None
        if fd is not None:
            os.close(fd)

    def array(self):
        """The mapping as a uint8 numpy array of nbytes (it keeps this object alive)."""
        return np.asarray(_View(self, self.nbytes))

    def register(self):
        import torch
        from . import _ffi
        dev = ctypes.c_void_p()
        device = torch.cuda.current_device()
        _ffi.call('teco_host_register', ctypes.c_void_p(self.addr), ctypes.c_size_t(self.size), ctypes.byref(dev))
        self._state['device'] = device
        self.dev_addr = int(dev.value)
        return self.dev_addr

    def close(self):
        self.close_fd()
        self.dev_addr = None
        self._finalizer()


def shared_mapping(nbytes, rank=0, world=1):
    """One HostMapping of `nbytes` per host, the same memory for every rank on that host, registered with the current
    device on each.  With world > 1 (an initialised torch.distributed group) the ranks are grouped by host name,
    gathered over the group; the lowest rank of each host creates the memfd and hands it to the others over an abstract
    socket whose name it gathers to them.  Returns (mapping, ranks on this host).  Any rank failing to create, share,
    map or register the memory raises HostStoreError on every rank, with every mapping released: the failures are
    gathered before each step that waits on another rank, so no rank is left waiting."""
    if world <= 1:
        m = None
        try:
            m = HostMapping.create(nbytes)
            m.close_fd()
            m.register()
        except (OSError, RuntimeError) as e:
            if m is not None:
                m.close()
            raise HostStoreError('the host frame store could not be set up: %s' % e) from e
        return m, (0,)
    import torch.distributed as dist

    def agree(why, got=None):
        out = [None] * world
        dist.all_gather_object(out, (why, got))
        whys = ['rank %d: %s' % (r, w) for r, (w, _) in enumerate(out) if w]
        if whys:
            if m is not None:
                m.close()
            raise HostStoreError('the host frame store could not be set up: ' + '; '.join(whys))
        return [g for _, g in out]
    hosts = [None] * world
    dist.all_gather_object(hosts, socket.gethostname())
    node = node_groups(hosts)[rank]
    lead = node[0] == rank
    sock = m = name = why = None
    try:
        if lead:
            m = HostMapping.create(nbytes)
            sock, name = fd_server(len(node) - 1)
            sock.settimeout(SHARE_TIMEOUT_S)
    except OSError as e:
        why = str(e)
    try:
        names = agree(why, name)
        why = None
        try:
            if lead:
                send_fd(sock, m.fd, len(node) - 1)
            else:
                m = HostMapping.from_fd(receive_fd(names[node[0]]), nbytes)
            m.register()
        except (OSError, RuntimeError) as e:
            why = str(e)
    finally:
        if sock is not None:
            sock.close()
        if m is not None:
            m.close_fd()
    agree(why)
    return m, node
