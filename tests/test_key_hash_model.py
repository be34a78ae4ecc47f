"""The numpy model of the key hash (keyhash.py) against the engine's own table on a host-only engine
(device=-1).  The GPU lookup tests build their collisions from this model: if it drifted from
hash.h they would build none and pass without testing anything, so this test must fail first."""
import pytest

from gpu_world import PCDN_ENOSPC
import keyhash as kh

SEEDS = [0, 0xF00DFACE12345679]
MAX_KEYS = 256                      # 128 buckets


def _engine(pcdn, seed, max_keys=MAX_KEYS):
    return pcdn.Engine(device=-1, max_conns=256, max_topics=16, max_keys=max_keys, max_key_len=64,
                       hash_seed=seed)


def test_model_matches_hash_h_reference_values():
    """fixed points of hash.h: the hash of the empty key is fmix64(0) == 0 (tag 1, bucket 0), and one
    non-trivial value computed by hand from the C++ definitions"""
    assert kh.key_hash(b"", 12345) == 0
    assert kh.place(b"", kh.DEFAULT_SEED, 128) == (1, 0, 0x5BD1E995 & 127)
    assert kh.n_buckets(1) == kh.n_buckets(2) == 1 and kh.n_buckets(3) == 2 and kh.n_buckets(256) == 128


@pytest.mark.parametrize("seed", SEEDS, ids=["builtin-seed", "top-bit-seed"])
def test_nine_keys_on_one_pair_are_refused_on_the_host(pcdn, seed):
    """Eight keys fill both buckets of a pair; the ninth finds no free slot anywhere on its walk and
    add_user fails with PCDN_ENOSPC, after which the other eight still resolve."""
    s, nb = kh.engine_seed(seed), kh.n_buckets(MAX_KEYS)
    p, keys = kh.full_pair(s, nb, 9)
    assert all(kh.pair(k, s, nb) == frozenset(p) for k in keys) and len(set(keys)) == 9
    e = _engine(pcdn, seed)
    conns = [e.add_user(k) for k in keys[:8]]
    with pytest.raises(pcdn.PcdnError) as ei:
        e.add_user(keys[8])
    assert ei.value.code == PCDN_ENOSPC
    assert [e.debug_route(k) for k in keys[:8]] == [(1, c) for c in conns]
    assert e.debug_route(keys[8]) == (0, -1)
    assert e.num_users()[0] == 8
    e.close()


@pytest.mark.parametrize("seed", SEEDS, ids=["builtin-seed", "top-bit-seed"])
def test_twins_resolve_to_their_own_connections_on_the_host(pcdn, seed):
    """Fingerprint twins (same tag, overlapping bucket pair; equal lengths and k / k + b"\\0") are
    both registered and each resolves to its own connection.  Six more keys on the twins' pair fill
    it: a seventh is refused, which shows that the engine puts both twins on that pair too."""
    s, nb = kh.engine_seed(seed), kh.n_buckets(MAX_KEYS)
    pairs = list(kh.twins(s, nb, 8, 2)) + list(kh.twins(s, nb, 21, 1))
    lt = kh.length_twin(s)
    pairs.append((lt, lt + b"\0"))
    for a, b in pairs:
        assert kh.is_twin(a, b, s, nb) and kh.pair(a, s, nb) == kh.pair(b, s, nb)
        fill = kh.keys_on_pair(s, nb, tuple(sorted(kh.pair(a, s, nb))), 7, 11)
        e = _engine(pcdn, seed)
        ca, cb = e.add_user(a), e.add_user(b)
        assert ca != cb
        assert e.debug_route(a) == (1, ca) and e.debug_route(b) == (1, cb)
        for k in fill[:6]:
            e.add_user(k)
        with pytest.raises(pcdn.PcdnError) as ei:
            e.add_user(fill[6])
        assert ei.value.code == PCDN_ENOSPC
        assert e.debug_route(a) == (1, ca) and e.debug_route(b) == (1, cb)
        e.remove_user(a)
        assert e.debug_route(a) == (0, -1) and e.debug_route(b) == (1, cb)
        e.close()
