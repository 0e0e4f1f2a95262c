"""Store family (ref surface: TCPStore.hpp:83-121 op list)."""
import os
import threading
import time

import pytest

from pytorch_distributed_train_b200 import _C


def _mk_tcp():
    master = _C.TCPStore("127.0.0.1", 0, -1, True, 5.0)
    client = _C.TCPStore("127.0.0.1", master.port, -1, False, 5.0)
    return master, client


@pytest.fixture(params=["hash", "tcp", "file", "prefix"])
def store(request, tmp_path):
    if request.param == "hash":
        yield _C.HashStore()
    elif request.param == "tcp":
        m, c = _mk_tcp()
        yield c
        del c, m
    elif request.param == "file":
        s = _C.FileStore(str(tmp_path / "fs"), 1)
        s.set_timeout(5.0)
        yield s
    else:
        base = _C.HashStore()
        yield _C.PrefixStore("pfx", base)


def test_set_get_add_cas(store):
    store.set("k", b"v1")
    assert store.get("k") == b"v1"
    assert store.add("ctr", 3) == 3
    assert store.add("ctr", -1) == 2
    assert store.get("ctr") == b"2"
    assert store.compare_set("new", "", "a") == b"a"
    assert store.compare_set("new", "zzz", "b") == b"a"
    assert store.compare_set("new", "a", "b") == b"b"
    assert store.check(["k", "ctr"]) and not store.check(["k", "nope"])
    assert store.delete_key("k") and not store.delete_key("k")
    store.append("ap", "x")
    store.append("ap", "yz")
    assert store.get("ap") == b"xyz"


def test_multi_and_queue(store):
    store.multi_set(["a", "b"], ["1", "2"])
    assert store.multi_get(["b", "a"]) == [b"2", b"1"]
    store.queue_push("q", "one")
    store.queue_push("q", "two")
    assert store.queue_len("q") == 2
    assert store.queue_pop("q") == b"one"
    assert store.queue_pop("q", False) == b"two"
    with pytest.raises(IndexError):
        store.queue_pop("q", False)


def test_wait_timeout_and_wakeup(store):
    t0 = time.time()
    with pytest.raises(TimeoutError):
        store.wait(["later"], 0.2)
    assert 0.15 < time.time() - t0 < 3.0
    threading.Timer(0.1, lambda: store.set("later", "x")).start()
    store.wait(["later"], 5.0)
    assert store.get("later") == b"x"


def test_get_blocks_until_set():
    m, c = _mk_tcp()
    got = []
    th = threading.Thread(target=lambda: got.append(c.get("slow")))
    th.start()
    time.sleep(0.1)
    assert th.is_alive()
    m.set("slow", "done")
    th.join(5)
    assert got == [b"done"]
    # a timed-out blocking call must not desynchronise the connection
    c.set_timeout(0.2)
    with pytest.raises(TimeoutError):
        c.get("never")
    c.set_timeout(5.0)
    c.set("after", "ok")
    assert c.get("after") == b"ok"


def test_concurrent_add_tcp():
    m, _ = _mk_tcp()
    clients = [_C.TCPStore("127.0.0.1", m.port, -1, False, 5.0) for _ in range(8)]

    def work(c):
        for _ in range(200):
            c.add("n", 1)

    ths = [threading.Thread(target=work, args=(c,)) for c in clients]
    [t.start() for t in ths]
    [t.join() for t in ths]
    assert m.add("n", 0) == 1600
    assert m.num_keys() >= 1


def test_master_waits_for_workers():
    port_box = []

    def master():
        s = _C.TCPStore("127.0.0.1", 0, 3, True, 10.0, False)
        port_box.append(s)

    master()
    m = port_box[0]
    ws = [_C.TCPStore("127.0.0.1", m.port, 3, False, 5.0) for _ in range(2)]
    assert m.add("__pdt_store_init__/workers", 0) == 3
    del ws


def test_client_connects_before_server_exists():
    import socket

    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        port = s.getsockname()[1]
    box = []
    th = threading.Thread(target=lambda: box.append(_C.TCPStore("127.0.0.1", port, -1, False, 5.0)))
    th.start()
    time.sleep(0.2)
    m = _C.TCPStore("127.0.0.1", port, -1, True, 5.0)
    th.join(5)
    assert box, "client should have retried until the server came up"
    m.set("x", "1")
    assert box[0].get("x") == b"1"


def test_store_barrier_reusable():
    m, _ = _mk_tcp()
    n = 4
    clients = [_C.TCPStore("127.0.0.1", m.port, -1, False, 5.0) for _ in range(n)]
    order = []

    def work(r):
        for it in range(3):
            _C.store_barrier(clients[r], "b", r, n, 5.0)
            order.append((it, r))

    ths = [threading.Thread(target=work, args=(r,)) for r in range(n)]
    [t.start() for t in ths]
    [t.join(10) for t in ths]
    its = [it for it, _ in order]
    assert its == sorted(its) and len(order) == 3 * n


def test_file_store_two_handles(tmp_path):
    p = str(tmp_path / "shared")
    a, b = _C.FileStore(p, 2), _C.FileStore(p, 2)
    a.set("k", "v")
    assert b.get("k") == b"v"
    assert b.add("c", 2) == 2 and a.add("c", 3) == 5
    assert os.path.exists(p)
