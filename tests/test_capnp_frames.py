"""Pins the hand-layout frame builder (capnp_frames.py): every frame meant to be valid decodes to the
intended (kind, field 0, field 1) through both the oracle's decoder and the engine's parser
(pcdn_parse_frame, the source k_parse runs on the device), and every frame meant to be malformed is
rejected by both.  Also: wire topic lists longer than 8192 entries on the host's Subscribe /
Unsubscribe path, which a host-only engine runs."""
import random

import pytest

import capnp_frames as cf
from oracle import oracle as orc

MAX_KEY = 128          # pcdn_config_default's max_key_len
CORPUS = cf.corpus(MAX_KEY)


def oracle_view(raw):
    """orc.deserialize as (kind, field 0, field 1) in the builder's terms, or None"""
    d = orc.deserialize(raw)
    if d is None:
        return None
    k, a, p = d
    return (k, p, b"") if k in (cf.USER_SYNC, cf.TOPIC_SYNC) else (k, a, p)


def engine_view(pcdn, raw):
    """(kind, field 0, topics as returned) from pcdn_parse_frame, or None on PCDN_EPARSE"""
    try:
        k, topics, (off, ln) = pcdn.parse_frame(raw)
    except pcdn.PcdnError as ex:
        assert ex.code == -7
        return None
    return k, raw[off:off + ln], topics


def test_corpus_covers_the_families():
    names = {n.split("/")[0] for n, _ in CORPUS}
    assert names == set(cf.FAMILIES) | set(cf.MALFORMED)
    for fam in cf.FAMILIES:
        assert all(cf.expected(s) is not None for n, s in CORPUS if n.startswith(fam + "/")), fam
    for fam in cf.MALFORMED:
        assert all(cf.expected(s) is None for n, s in CORPUS if n.startswith(fam + "/")), fam
    lay = {fam: cf.build(cf.family_spec(fam, cf.DIRECT, b"k" * 9, b"m" * 17))[1] for fam in cf.FAMILIES}
    assert len(lay["segs-511"].segs) == 511 and len(lay["segs-odd"].segs) == 3 and len(lay["segs-even-pad"].segs) == 2
    assert len(lay["all-dfar"].segs) == 9       # 4 objects, each with a pad segment of its own
    assert len(cf.build(cf.family_spec("segs-512", cf.DIRECT, b"", b""))[1].segs) == 512
    # the list that claims one word past its segment: that word is the next segment's, inside the frame,
    # so only a bound by the segment (not by the frame) rejects it
    for n in (0, 8, 9):
        raw, lay = cf.build(cf.family_spec("f0-over-into-next-segment", cf.BROADCAST, bytes(n), b"m"))
        assert len(lay.segs) == 3 and len(lay.segs[2]) > 0
        assert lay.offset(1, len(lay.segs[1])) + 8 <= len(raw)


@pytest.mark.parametrize("kind,f0,f1", [(cf.DIRECT, b"", b""), (cf.DIRECT, b"key-0123", b"m" * 100),
                                        (cf.BROADCAST, bytes([1, 2, 2, 9]), b"x" * 7),
                                        (cf.SUBSCRIBE, bytes([3]), b""), (cf.UNSUBSCRIBE, bytes(range(9)), b""),
                                        (cf.USER_SYNC, b"blob" * 5, b"")])
def test_near_layout_is_the_oracle_encoding(kind, f0, f1):
    """the default spec lays a small message out byte for byte as the reference's encoder does"""
    want = orc.serialize(kind, b"", f0) if kind == cf.USER_SYNC else orc.serialize(kind, f0, f1)   # a sync blob is the payload there
    assert cf.frame(cf.Spec(kind, f0, f1)) == want


@pytest.mark.parametrize("name,spec", CORPUS, ids=[n for n, _ in CORPUS])
def test_frame_decodes_as_intended(pcdn, name, spec):
    raw = cf.frame(spec)
    want = cf.expected(spec)
    got_o = oracle_view(raw)
    got_e = engine_view(pcdn, raw)
    if want is None:
        assert got_o is None and got_e is None
        return
    assert got_o == want
    k, f0, topics = got_e
    assert (k, f0) == want[:2]
    if k in (cf.BROADCAST, cf.SUBSCRIBE, cf.UNSUBSCRIBE):
        assert topics == list(want[1][:256])


def test_mutated_frames_agree():
    """structure-aware mutations of the whole corpus: the oracle and the builder's layout marks stay
    in step (every mutated frame is decoded by the oracle without a crash, and some of every family
    survive as valid frames)"""
    rng = random.Random(5)
    alive = set()
    for name, spec in CORPUS[::3]:
        raw, lay = cf.build(spec)
        for _ in range(3):
            m = cf.mutate(rng, raw, lay)
            assert len(m) == len(raw)
            if oracle_view(m) is not None:
                alive.add(name.split("/")[0])
    assert len(alive) > len(cf.FAMILIES) // 2


def test_mutated_frames_parse_like_the_oracle(pcdn):
    rng = random.Random(6)
    n_valid = 0
    for name, spec in CORPUS:
        raw, lay = cf.build(spec)
        m = cf.mutate(rng, raw, lay)
        o, e = oracle_view(m), engine_view(pcdn, m)
        assert (o is None) == (e is None), name
        if o is not None:
            n_valid += 1
            assert e[0] == o[0] and e[1] == o[1], name
    assert n_valid > len(CORPUS) // 10


@pytest.mark.parametrize("kind", [cf.SUBSCRIBE, cf.UNSUBSCRIBE])
@pytest.mark.parametrize("n_valid", [0, 12])
@pytest.mark.parametrize("n", [8191, 8192, 8193, 9000, 20000])
def test_long_topic_list_subscribe(pcdn, kind, n_valid, n):
    """a Subscribe / Unsubscribe whose wire list is longer than 8192 entries is pruned and applied as
    the reference applies it (no length limit), whether it prunes to one topic or keeps them all"""
    e = pcdn.Engine(device=-1, max_conns=64, max_topics=256, max_keys=64, n_valid_topics=n_valid)
    o = orc.Oracle("/", n_valid)
    key = b"u" * 8
    c = e.add_user(key, [3, 5] if kind == cf.UNSUBSCRIBE else [])
    o.add_user(key, [3, 5] if kind == cf.UNSUBSCRIBE else [])
    for topics in ([3] * n, [3, 5] * (n // 2) + [3] * (n % 2), [3] + [200] * (n - 1)):
        raw = cf.frame(cf.Spec(kind, bytes(topics)))
        want = o.user_receive(key, raw)
        assert want in (0, -8)
        assert e.user_receive(key, raw) == want, pcdn.lib().pcdn_last_error()
        for t in (3, 5, 200):
            assert (c in e.debug_interested([t])) == (o.user_conn(key) in o.interested([t])), (topics[:4], t)
    e.close()
