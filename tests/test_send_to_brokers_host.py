"""pcdn_send_to_broker / pcdn_send_to_brokers without a GPU: the restatement of Inner::try_send_to_broker /
try_send_to_brokers (cdn-broker/src/tasks/broker/sender.rs:17-59, in gpu_world.py) on the oracle that the GPU tests
compare against, the host-only engine's answer and the argument checks that come before it."""
import ctypes as C

import pytest

from gpu_world import PCDN_EINVAL, PCDN_ENODEV, try_send_to_broker, try_send_to_brokers
from oracle import oracle as orc


def framed(raw):
    return len(raw).to_bytes(4, "big") + raw


@pytest.fixture
def sync_frames():
    """a UserSync and a TopicSync message as the host builds them (the engine never parses them)"""
    return (orc.serialize(orc.KIND_USER_SYNC, b"", b"user-sync archive" * 7),
            orc.serialize(orc.KIND_TOPIC_SYNC, b"", b"topic-sync archive" * 3))


def test_oracle_sends_to_one_broker_and_to_every_broker(sync_frames):
    us, ts = sync_frames
    o = orc.Oracle("/")
    user = o.add_user(b"u" * 32, [0, 1])
    a, b, c = o.add_broker("a/a"), o.add_broker("b/b"), o.add_broker("c/c")
    o.subscribe_broker_to("a/a", [0])          # subscriptions play no part
    assert try_send_to_broker(o, "b/b", ts) == 0
    assert try_send_to_brokers(o, ["a/a", "b/b", "c/c"], us) == 0
    assert o.stream(a) == framed(us)
    assert o.stream(b) == framed(ts) + framed(us)
    assert o.stream(c) == framed(us)
    assert o.stream(user) == b""               # users never get these frames
    assert o.deliveries() == 4 and o.bytes_sent() == len(ts) + 3 * len(us)


def test_oracle_unknown_identifier_and_no_broker(sync_frames):
    us, _ = sync_frames
    o = orc.Oracle("/")
    user = o.add_user(b"u" * 32, [0])
    assert try_send_to_brokers(o, [], us) == 1          # the loop over no broker (sender.rs:52-57)
    a = o.add_broker("a/a")
    assert try_send_to_broker(o, "x/x", us) == 1        # if let Some(connection) (sender.rs:29)
    assert try_send_to_brokers(o, ["x/x"], us) == 1
    assert o.stream(a) == b"" and o.stream(user) == b"" and o.deliveries() == 0


def test_oracle_removed_broker_and_kick(sync_frames):
    us, ts = sync_frames
    o = orc.Oracle("/")
    a, b = o.add_broker("a/a"), o.add_broker("b/b")
    o.remove_broker("a/a")
    assert try_send_to_broker(o, "a/a", us) == 1
    assert try_send_to_brokers(o, ["a/a", "b/b"], ts) == 0
    assert o.stream(a) == b"" and o.stream(b) == framed(ts)
    b2 = o.add_broker("b/b")                   # same identifier again: the old connection is kicked
    assert b2 != b and o.conn_removed(b)
    assert try_send_to_broker(o, "b/b", us) == 0
    assert o.stream(b) == framed(ts) and o.stream(b2) == framed(us)
    assert o.num_users() == 0                           # the relay keys are no users


def test_host_only_engine_refuses_with_enodev(pcdn, sync_frames):
    us, _ = sync_frames
    e = pcdn.Engine(device=-1)
    e.add_broker("a/a")
    for call in (lambda: e.send_to_broker("a/a", us), lambda: e.send_to_brokers(us)):
        with pytest.raises(pcdn.PcdnError) as ei:
            call()
        assert ei.value.code == PCDN_ENODEV
        assert "host-only" in e.L.pcdn_last_error().decode()
    e.close()


def test_bad_arguments(pcdn):
    e = pcdn.Engine(device=-1)
    e.add_broker("a/a")
    L = e.L
    assert L.pcdn_send_to_brokers(e.h, None, 5) == PCDN_EINVAL
    assert "null frame" in L.pcdn_last_error().decode()
    assert L.pcdn_send_to_broker(e.h, b"a/a", None, 1) == PCDN_EINVAL
    buf = C.create_string_buffer(16)
    # longer than MAX_MESSAGE_SIZE (cdn-proto/src/lib.rs:25): refused before the frame is read
    assert L.pcdn_send_to_brokers(e.h, C.cast(buf, C.c_char_p), 0x20000000) == PCDN_EINVAL
    assert "MAX_MESSAGE_SIZE" in L.pcdn_last_error().decode()
    assert L.pcdn_send_to_broker(e.h, None, C.cast(buf, C.c_char_p), 0x20000000) == PCDN_EINVAL
    e.close()
