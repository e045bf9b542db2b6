"""Control plane: ``Master`` (rendezvous KV tree), ``MasterClient`` and the ``Server`` shim.

Reference: the TCP master is a single-thread poll() KV tree with ephemeral nodes and
watchers (pico-core rpc/Master.cpp:139-304); ``MasterClient`` offers tree_node_*, barrier,
acquire/release_lock, generate_id and the rpc/node/model registries
(rpc/MasterClient.h:56-160); ``Server`` joins a job as a dedicated PS process
(openembedding/entry/server.cc:25-60, py_api.cc:164-215).

Design: inside one NVSwitch box every rank hosts its own shards in HBM, so training
needs no server process and no data-plane RPC. The control plane keeps the same verbs on top
of a ``torch.distributed.TCPStore`` (the store server thread plays the master): tree paths
are store keys, children are tracked in an append-only per-parent index, ephemeral nodes are
heartbeat leases (a node whose lease is older than ``LEASE_S`` is dead -- the reference drops
them on socket close, Master.cpp:203). Watchers (Master.cpp:247-304 notifies the registered
connections of a node and of its parent): every mutation bumps a version counter of the node
and of its parent and creates the notification key of that version; a watcher blocks in the
store's server-side ``wait`` on the NEXT version's key (its own connection), so a change wakes
it without polling.
"""
import datetime
import socket
import threading
import time
import uuid

LEASE_S = 5.0
_TOMB = "\x00deleted"


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    return port


class Master:
    """In-process master; ``endpoint`` is what workers put in ``flags.master_endpoint``."""

    def __init__(self, bind_ip="127.0.0.1", port=0):
        from torch.distributed import TCPStore
        self.ip = bind_ip or "127.0.0.1"
        self.port = port or _free_port()
        self._store = TCPStore(self.ip, self.port, is_master=True, wait_for_workers=False,
                               timeout=datetime.timedelta(seconds=3600))

    @property
    def endpoint(self):
        return "%s:%d" % (self.ip, self.port)

    def client(self, **kw):
        return MasterClient(self.endpoint, **kw)

    def finalize(self):
        self._store = None

    join = finalize


class MasterClient:
    """Tree / barrier / lock / id verbs (pico-core rpc/MasterClient.h:56-160)."""

    def __init__(self, endpoint, root_path="/openembedding", timeout=3600):
        from torch.distributed import TCPStore
        ip, port = endpoint.rsplit(":", 1)
        self.endpoint = endpoint
        self.root = "/" + root_path.strip("/")
        self._store = TCPStore(ip, int(port), is_master=False, timeout=datetime.timedelta(seconds=timeout))
        self._session = uuid.uuid4().hex
        self._leases = {}
        self._hb = None
        self._stop = threading.Event()
        self._my_watches = []

    # ---- key helpers
    def _norm(self, path):
        return "/" + path.strip("/") if path.strip("/") else ""

    def _vk(self, path):
        return "v:" + self.root + self._norm(path)

    def _ik(self, path):
        return "i:" + self.root + self._norm(path)

    def _get(self, key):
        if not self._store.check([key]):
            return None
        v = self._store.get(key).decode()
        return None if v == _TOMB else v

    def _index_child(self, path):
        p = self._norm(path)
        if not p:
            return
        parent, _, name = p.rpartition("/")
        self._store.append(self._ik(parent), name + "\n")

    # ---- change notification
    def _wk(self, path):
        return "w:" + self.root + self._norm(path)

    def _notify(self, path):
        """bump the version of `path` and of its parent and publish the notification keys of the new versions"""
        p = self._norm(path)
        targets = [p]
        if p:
            targets.append(p.rpartition("/")[0])
        for t in targets:
            ver = int(self._store.add("w:" + self.root + t, 1))
            self._store.set("n:" + self.root + t + "#%d" % ver, "1")
            if ver > 2:
                try:
                    self._store.delete_key("n:" + self.root + t + "#%d" % (ver - 2))
                except Exception:
                    pass

    def node_version(self, path):
        """number of changes of `path` or of one of its children so far"""
        return int(self._store.add(self._wk(path), 0))

    def watch(self, path, callback, poll_s=0.5):
        """call ``callback(path, version)`` (on a watcher thread) after every change of `path` or of one of its direct
        children -- add, set, delete, or an ephemeral child created / removed. Returns a handle with ``cancel()``.
        The thread blocks server-side on the notification key of the next version (its own store connection)."""
        return _Watch(self, path, callback, poll_s)

    # ---- tree
    def tree_node_add(self, path, value="", ephemeral=False):
        """create; False if the node already exists"""
        key = self._vk(path)
        cur = self._store.compare_set(key, "", value if value else " ").decode()
        ok = cur == (value if value else " ")
        if not ok and cur == _TOMB:
            cur = self._store.compare_set(key, _TOMB, value if value else " ").decode()
            ok = cur == (value if value else " ")
        if ok:
            self._index_child(path)
            if ephemeral:
                self._lease(path)
            self._notify(path)
        return ok

    def tree_node_set(self, path, value):
        existed = self._get(self._vk(path)) is not None
        self._store.set(self._vk(path), value if value else " ")
        if not existed:
            self._index_child(path)
        self._notify(path)
        return True

    def tree_node_get(self, path, default=None):
        v = self._get(self._vk(path))
        if v is None or not self._alive(path):
            return default
        return "" if v == " " else v

    def tree_node_del(self, path):
        if self._get(self._vk(path)) is None:
            return False
        self._store.set(self._vk(path), _TOMB)
        self._leases.pop(self._norm(path), None)
        self._notify(path)
        return True

    def tree_node_sub(self, path):
        """names of the live children of `path`"""
        ik = self._ik(path)
        if not self._store.check([ik]):
            return []
        names = sorted(set(n for n in self._store.get(ik).decode().split("\n") if n))
        base = self._norm(path)
        return [n for n in names if self._get(self._vk(base + "/" + n)) is not None and self._alive(base + "/" + n)]

    # ---- ephemeral nodes = heartbeat leases
    def _lk(self, path):
        return "l:" + self.root + self._norm(path)

    def _lease(self, path):
        self._leases[self._norm(path)] = True
        self._store.set(self._lk(path), repr(time.time()))
        if self._hb is None:
            self._hb = threading.Thread(target=self._beat, daemon=True)
            self._hb.start()

    def _beat(self):
        while not self._stop.wait(LEASE_S / 3):
            for p in list(self._leases):
                try:
                    self._store.set(self._lk(p), repr(time.time()))
                except Exception:
                    return

    def _alive(self, path):
        lk = self._lk(path)
        if not self._store.check([lk]):
            return True          # not ephemeral
        return time.time() - float(self._store.get(lk).decode()) < LEASE_S

    def close(self):
        self._stop.set()
        for w in list(self._my_watches):
            w.cancel(join=True)
        self._my_watches = []

    # ---- ids / barriers / locks
    def generate_id(self, name):
        return int(self._store.add("id:" + self.root + "/" + name, 1)) - 1

    def advance_counter(self, name, by):
        """atomically add `by` to a cluster-wide counter; returns its value BEFORE the addition (fetch_add)"""
        by = int(by)
        return int(self._store.add("c:" + self.root + "/" + name, by)) - by

    def barrier(self, name, n, timeout=3600):
        key = "b:" + self.root + "/" + name
        arrived = int(self._store.add(key, 1))
        target = ((arrived - 1) // n + 1) * n
        t0 = time.time()
        while int(self._store.add(key, 0)) < target:
            if time.time() - t0 > timeout:
                raise TimeoutError("master barrier " + name)
            time.sleep(0.002)

    def acquire_lock(self, name, timeout=3600):
        key = "k:" + self.root + "/" + name
        t0 = time.time()
        while True:
            for expected in ("", "free"):
                if self._store.compare_set(key, expected, self._session).decode() == self._session:
                    return
            if time.time() - t0 > timeout:
                raise TimeoutError("master lock " + name)
            time.sleep(0.002)

    def release_lock(self, name):
        self._store.set("k:" + self.root + "/" + name, "free")


_watches = []


def _cancel_watches():
    """interpreter exit: no watcher thread may still sit inside the store client when it is torn down"""
    for w in list(_watches):
        w.cancel(join=True)


import atexit  # noqa: E402
atexit.register(_cancel_watches)


class _Watch:
    """one watcher: a thread with its own store connection, blocked in ``wait`` on the next version's key"""

    def __init__(self, client, path, callback, poll_s):
        from torch.distributed import TCPStore
        ip, port = client.endpoint.rsplit(":", 1)
        self._store = TCPStore(ip, int(port), is_master=False, timeout=datetime.timedelta(seconds=3600))
        self._prefix = "n:" + client.root + client._norm(path) + "#"
        self._wk = client._wk(path)
        self.path, self.callback, self.poll_s = path, callback, poll_s
        self.version = int(self._store.add(self._wk, 0))
        self._stop = threading.Event()
        self._t = threading.Thread(target=self._run, daemon=True)
        _watches.append(self)
        client._my_watches.append(self)
        self._t.start()

    def _run(self):
        while not self._stop.is_set():
            try:
                self._store.wait([self._prefix + "%d" % (self.version + 1)], datetime.timedelta(seconds=self.poll_s))
            except Exception:
                # timeout: nothing yet (or several versions went by at once and the key was collected): resync below
                pass
            if self._stop.is_set():
                return
            try:
                cur = int(self._store.add(self._wk, 0))
            except Exception:
                return
            if cur != self.version:
                self.version = cur
                try:
                    self.callback(self.path, cur)
                except Exception:
                    pass

    def cancel(self, join=False):
        self._stop.set()
        if self in _watches:
            _watches.remove(self)
        if join and self._t.is_alive() and threading.current_thread() is not self._t:
            self._t.join(self.poll_s + 1.0)


class Server:
    """Standalone shard host for serving (``serving.node.ServingNode`` in a thread).

    Training on one box never needs it: ``flags.wait_num_servers == -1`` (each worker hosts
    its shards in its own HBM) is the only training topology.
    """

    def __init__(self, master_endpoint="", bind_ip="127.0.0.1", config="", port=0):
        from .serving.node import ServingNode
        self._node = ServingNode(master_endpoint=master_endpoint, bind_ip=bind_ip, config=config, port=port)
        self._thread = threading.Thread(target=self._node.serve_forever, daemon=True)
        self._thread.start()

    @property
    def endpoint(self):
        return self._node.endpoint

    @property
    def node_id(self):
        return self._node.node_id

    def exit(self):
        self._node.shutdown()

    def join(self):
        self._thread.join()


def main(argv=None):
    """``python -m openembedding_b200.master --bind_ip 0.0.0.0 --port 9090`` -- the standalone master
    (reference: ``masterd``, pico-ps/pico-core/src/masterd.cc / openembedding/entry/masterd.cc)."""
    import argparse
    import signal
    ap = argparse.ArgumentParser(prog="masterd")
    ap.add_argument("--bind_ip", "--rpc_bind_ip", dest="bind_ip", default="127.0.0.1")
    ap.add_argument("--port", type=int, default=0)
    ap.add_argument("--endpoint", default="", help="ip:port (overrides --bind_ip/--port)")
    a = ap.parse_args(argv)
    ip, port = a.bind_ip, a.port
    if a.endpoint:
        ip, p = a.endpoint.rsplit(":", 1)
        port = int(p)
    m = Master(ip, port)
    print("master endpoint %s" % m.endpoint, flush=True)
    stop = threading.Event()
    for sig in (signal.SIGINT, signal.SIGTERM):
        signal.signal(sig, lambda *_: stop.set())
    stop.wait()
    m.finalize()


if __name__ == "__main__":
    main()
