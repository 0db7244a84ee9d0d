"""CPU: the host rings a data rank without a GPU exchanges micro-batches and results through - two processes over a
socketpair and one POSIX shared-memory segment, both ends through the host-only entry points (`pe_hostring_*`):
order across many wrap-arounds, back-pressure, close, header checks, oversized payloads, the segment's lifetime and the
bounded waits."""
import ctypes
import os
import signal
import socket
import threading
import time
import pytest

from pipeedge_b200._lib import LIB, PipeEdgeB200Error, check

SLOTS = 3
ROOM = 4096 * 3           # payload bytes per slot the producer asks for


def _name(tag):
    return f"/pipeedge_b200_test_{os.getpid()}_{tag}"


def _payload(i):
    """Payload i: 1..ROOM bytes (not all multiples of 16), items 1..8, a pattern that names i."""
    n = 1 + (i * 977) % ROOM
    return bytes((i * 31 + j) & 0xff for j in range(n)), 1 + i % 8


def _create(sock, name, is_producer):
    handle = ctypes.c_void_p()
    check(LIB.pe_hostring_create(sock.fileno(), name.encode(), 1 if is_producer else 0, ROOM if is_producer else 0,
                                 SLOTS if is_producer else 0, ctypes.byref(handle)))
    return handle


def _attach(sock, is_producer):
    handle = ctypes.c_void_p()
    check(LIB.pe_hostring_attach(sock.fileno(), 1 if is_producer else 0, ROOM if is_producer else 0,
                                 SLOTS if is_producer else 0, ctypes.byref(handle)))
    return handle


def _publish_all(ring, count):
    for i in range(count):
        data, items = _payload(i)
        check(LIB.pe_hostring_publish(ring, data, len(data), items, i))
    check(LIB.pe_hostring_close_input(ring))


def _drain(ring):
    """Every payload until the close: [(ticket, bytes)]."""
    got = []
    ticket = (ctypes.c_longlong * 2)()
    data = ctypes.c_void_p()
    while True:
        rc = LIB.pe_hostring_next(ring, ticket)
        if rc == 1:
            return got
        check(rc)
        items, index = int(ticket[0]), int(ticket[1])
        want, _ = _payload(index)
        check(LIB.pe_hostring_wait(ring, items, len(want), ctypes.byref(data)))
        got.append(((items, index), ctypes.string_at(data.value, len(want))))
        check(LIB.pe_hostring_release(ring))


def _fork(fn):
    """Run fn() in a forked child (ctypes calls only) that exits with 0 on success, 1 on an exception."""
    pid = os.fork()
    if pid == 0:
        code = 1
        try:
            fn()
            code = 0
        finally:
            os._exit(code)   # pylint: disable=protected-access
    return pid


def _join(pid):
    _, status = os.waitpid(pid, 0)
    return status


@pytest.mark.parametrize('creator_produces', [True, False])
def test_bytes_round_trip_in_order_over_many_wrap_arounds(creator_produces):
    """The data rank creates the segment as the producer (its inputs) or the consumer (its results); 10 R payloads of
    varying sizes and item counts arrive in order, byte for byte; the close reaches the consumer; nothing is left in
    /dev/shm."""
    name = _name(f"rt{int(creator_produces)}")
    a, b = socket.socketpair()
    count = 10 * SLOTS + 1

    def child():
        ring = _attach(b, not creator_produces)
        if creator_produces:
            got = _drain(ring)
            assert [t for t, _ in got] == [(_payload(i)[1], i) for i in range(count)]
            assert all(data == _payload(i)[0] for i, (_, data) in enumerate(got))
        else:
            _publish_all(ring, count)
        LIB.pe_hostring_close(ring)

    pid = _fork(child)
    try:
        ring = _create(a, name, creator_produces)
        assert not os.path.exists('/dev/shm' + name), "the segment outlived the handshake"
        assert LIB.pe_hostring_slot_bytes(ring) >= ROOM
        if creator_produces:
            _publish_all(ring, count)
        else:
            got = _drain(ring)
            assert [t for t, _ in got] == [(_payload(i)[1], i) for i in range(count)]
            assert all(data == _payload(i)[0] for i, (_, data) in enumerate(got))
        LIB.pe_hostring_close(ring)
    finally:
        assert _join(pid) == 0
        a.close()
        b.close()


def test_producer_blocks_until_a_slot_is_released():
    """R payloads go out without a release; the next publish waits until the consumer releases one, then completes."""
    name = _name('bp')
    a, b = socket.socketpair()
    gate_r, gate_w = os.pipe()

    def child():
        ring = _attach(b, False)
        ticket = (ctypes.c_longlong * 2)()
        data = ctypes.c_void_p()
        for i in range(SLOTS + 1):
            check(LIB.pe_hostring_next(ring, ticket))
            want, items = _payload(i)
            check(LIB.pe_hostring_wait(ring, items, len(want), ctypes.byref(data)))
            assert ctypes.string_at(data.value, len(want)) == want
            if i == 0:
                os.read(gate_r, 1)   # hold the first slot until the parent has seen the producer blocked
            check(LIB.pe_hostring_release(ring))
        assert LIB.pe_hostring_next(ring, ticket) == 1
        LIB.pe_hostring_close(ring)

    pid = _fork(child)
    try:
        ring = _create(a, name, True)
        for i in range(SLOTS):
            data, items = _payload(i)
            check(LIB.pe_hostring_publish(ring, data, len(data), items, i))
        data, items = _payload(SLOTS)
        rcs = []
        thr = threading.Thread(target=lambda: rcs.append(LIB.pe_hostring_publish(ring, data, len(data), items, SLOTS)))
        thr.start()
        time.sleep(0.5)
        assert thr.is_alive() and not rcs, "the producer overwrote a slot the consumer had not released"
        os.write(gate_w, b'x')
        thr.join(10)
        assert rcs == [0]
        check(LIB.pe_hostring_close_input(ring))
        LIB.pe_hostring_close(ring)
    finally:
        assert _join(pid) == 0
        for fd in (gate_r, gate_w):
            os.close(fd)
        a.close()
        b.close()


def test_mismatched_headers_and_oversized_payloads_are_refused():
    """A consumer expecting other items or another size, or finding a header whose magic is not a link's, is refused
    (and may wait again); a payload larger than a slot is refused before anything is written or announced."""
    name = _name('hdr')
    a, b = socket.socketpair()

    def child():
        ring = _attach(b, True)
        room = LIB.pe_hostring_slot_bytes(ring)
        big = b'\0' * (room + 1)
        assert LIB.pe_hostring_publish(ring, big, len(big), 1, 0) != 0
        assert b'exceed' in LIB.pe_last_error()
        check(LIB.pe_hostring_publish(ring, b'abcdefgh' * 4, 32, 2, 7))
        check(LIB.pe_hostring_close_input(ring))
        LIB.pe_hostring_close(ring)

    pid = _fork(child)
    try:
        ring = _create(a, name, False)
        ticket = (ctypes.c_longlong * 2)()
        data = ctypes.c_void_p()
        check(LIB.pe_hostring_next(ring, ticket))
        assert list(ticket) == [2, 7]   # the oversized payload never announced itself
        for items, nbytes in ((3, 32), (2, 31), (2, 33)):
            with pytest.raises(PipeEdgeB200Error, match='mismatch'):
                check(LIB.pe_hostring_wait(ring, items, nbytes, ctypes.byref(data)))
        check(LIB.pe_hostring_wait(ring, 2, 32, ctypes.byref(data)))
        assert ctypes.string_at(data.value, 32) == b'abcdefgh' * 4
        magic = ctypes.c_uint32.from_address(data.value - 16384)
        good = magic.value
        magic.value = good ^ 1
        with pytest.raises(PipeEdgeB200Error, match='mismatch'):
            check(LIB.pe_hostring_wait(ring, 2, 32, ctypes.byref(data)))
        magic.value = good
        check(LIB.pe_hostring_release(ring))
        assert LIB.pe_hostring_next(ring, ticket) == 1
        LIB.pe_hostring_close(ring)
    finally:
        assert _join(pid) == 0
        a.close()
        b.close()


def test_no_segment_is_left_when_the_peer_dies_during_the_handshake():
    """The stage's process dies after the data rank has created the segment and offered it: the handshake fails on
    the data rank and the segment is gone."""
    name = _name('kill')
    a, b = socket.socketpair()

    def child():
        b.recv(1)                                 # the hello has arrived: the segment exists
        os.kill(os.getpid(), signal.SIGKILL)

    pid = _fork(child)
    b.close()
    try:
        handle = ctypes.c_void_p()
        rc = LIB.pe_hostring_create(a.fileno(), name.encode(), 1, ROOM, SLOTS, ctypes.byref(handle))
        assert rc != 0 and b"the consumer's reply" in LIB.pe_last_error()   # closed or reset
        assert not os.path.exists('/dev/shm' + name)
    finally:
        assert os.WIFSIGNALED(_join(pid))
        a.close()


def test_a_peer_that_never_answers_ends_in_the_bounded_wait_error(monkeypatch):
    """No reply to the offer; then, on a ring whose consumer never releases, a publish beyond R: both end in the
    link-timeout error instead of hanging, and no segment is left."""
    monkeypatch.setenv('PIPEEDGE_LINK_TIMEOUT_S', '0.5')
    name = _name('mute')
    a, b = socket.socketpair()
    try:
        handle = ctypes.c_void_p()
        t0 = time.monotonic()
        rc = LIB.pe_hostring_create(a.fileno(), name.encode(), 1, ROOM, SLOTS, ctypes.byref(handle))
        assert rc != 0 and b'within the link timeout' in LIB.pe_last_error()
        assert time.monotonic() - t0 < 10
        assert not os.path.exists('/dev/shm' + name)
    finally:
        a.close()
        b.close()

    a, b = socket.socketpair()
    gate_r, gate_w = os.pipe()

    def child():
        ring = _attach(b, False)
        os.read(gate_r, 1)   # never reads a payload, never releases
        LIB.pe_hostring_close(ring)

    pid = _fork(child)
    try:
        ring = _create(a, name, True)
        for i in range(SLOTS):
            check(LIB.pe_hostring_publish(ring, b'x' * 64, 64, 1, i))
        t0 = time.monotonic()
        assert LIB.pe_hostring_publish(ring, b'x' * 64, 64, 1, SLOTS) != 0
        assert b'did not release' in LIB.pe_last_error()
        assert 0.4 < time.monotonic() - t0 < 10
        LIB.pe_hostring_close(ring)
    finally:
        os.write(gate_w, b'x')
        assert _join(pid) == 0
        for fd in (gate_r, gate_w):
            os.close(fd)
        a.close()
        b.close()
