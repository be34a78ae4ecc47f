"""numpy model of the direct-map key hash (push-cdn_b200/csrc/hash.h) and generators of the keys
where a partial-key cuckoo lookup can go wrong: many keys on one bucket pair, and fingerprint twins
(two keys with the same tag whose bucket pairs overlap, so a lookup of one sees the other as a
candidate and only the full-key compare tells them apart).

The hash is a sum of per-word mixes, so the generators vary only the first 64-bit word of a key and
keep the others fixed: the fixed words add a constant to the sum.  ``tests/test_key_hash_model.py``
pins the model against a host-only engine; the GPU tests build their collisions from it.
"""
from __future__ import annotations

import functools

import numpy as np

DEFAULT_SEED = 0x243F6A8885A308D3   # pcdn_config.hash_seed == 0 selects this one
M64 = (1 << 64) - 1
_U = np.uint64


def engine_seed(hash_seed: int) -> int:
    return hash_seed if hash_seed else DEFAULT_SEED


def n_buckets(max_keys: int) -> int:
    """the engine's table size: 4-slot buckets, load factor <= 50 %"""
    nb = 1
    while nb * 2 < max_keys:
        nb <<= 1
    return nb


def fmix64(k):
    k = np.asarray(k, dtype=np.uint64)
    k = k ^ (k >> _U(33))
    k = k * _U(0xFF51AFD7ED558CCD)
    k = k ^ (k >> _U(33))
    k = k * _U(0xC4CEB9FE1A85EC53)
    return k ^ (k >> _U(33))


def key_word_mix(w, i: int, seed: int):
    return fmix64(np.asarray(w, dtype=np.uint64) ^ _U((seed + (i + 1) * 0x9E3779B97F4A7C15) & M64))


def key_hash_finish(acc, length: int):
    return fmix64(np.asarray(acc, dtype=np.uint64) ^ _U((length * 0xD6E8FEB86659FD93) & M64))


def key_tag(h):
    return ((np.asarray(h, dtype=np.uint64) >> _U(32)) | _U(1)).astype(np.uint32)


def key_bucket(h, nb: int):
    return (np.asarray(h, dtype=np.uint64) & _U(nb - 1)).astype(np.uint32)


def alt_bucket(b, tag, nb: int):
    prod = (np.asarray(tag, dtype=np.uint64) * _U(0x5BD1E995)) & _U(0xFFFFFFFF)
    return ((np.asarray(b, dtype=np.uint64) ^ prod) & _U(nb - 1)).astype(np.uint32)


def _words(key: bytes):
    pad = key + bytes(-len(key) % 8)
    return [int.from_bytes(pad[i:i + 8], "little") for i in range(0, len(pad), 8)]


def key_hash(key: bytes, seed: int) -> int:
    """the hash of one key (hash.h key_hash_host), `seed` as the engine uses it (engine_seed)"""
    with np.errstate(over="ignore"):
        acc = np.zeros(1, dtype=np.uint64)
        for i, w in enumerate(_words(key)):
            acc = acc + key_word_mix(np.array([w], dtype=np.uint64), i, seed)
        return int(key_hash_finish(acc, len(key))[0])


def place(key: bytes, seed: int, nb: int):
    """(tag, b1, b2) of a key in a table of `nb` buckets"""
    h = key_hash(key, seed)
    tag = int(key_tag(h))
    b1 = int(key_bucket(h, nb))
    return tag, b1, int(alt_bucket(b1, tag, nb))


def pair(key: bytes, seed: int, nb: int):
    _, b1, b2 = place(key, seed, nb)
    return frozenset((b1, b2))


# ---------------------------------------------------------------- candidate keys (first word varies)
def _candidates(seed: int, length: int, start: int, count: int, fill: int):
    """keys of `length` bytes: word 0 = a bijective scramble of start..start+count-1 (kept to the key's
    bytes), every other byte `fill`.  Returns (word 0 of every key, its hash); _key rebuilds a key."""
    assert length >= 3, "too few bytes in the first word to search over"
    lw = min(length, 8)
    idx = np.arange(start, start + count, dtype=np.uint64)
    with np.errstate(over="ignore"):
        w0 = (idx * _U(0x2545F4914F6CDD1D)) & _U((1 << (8 * lw)) - 1)
        tail = _words(bytes(8) + bytes([fill]) * (length - 8)) if length > 8 else [0]
        const = 0
        for i, w in enumerate(tail[1:], start=1):
            const = (const + int(key_word_mix(np.array([w], dtype=np.uint64), i, seed)[0])) & M64
        h = key_hash_finish(key_word_mix(w0, 0, seed) + _U(const), length)
    return w0, h


def _key(w0: int, length: int, fill: int) -> bytes:
    lw = min(length, 8)
    return int(w0).to_bytes(8, "little")[:lw] + bytes([fill]) * (length - lw)


@functools.lru_cache(maxsize=None)
def keys_on_pair(seed: int, nb: int, buckets: tuple, n: int, length: int = 8, fill: int = 0x5A, first=None):
    """`n` keys of `length` bytes whose bucket pair is exactly {buckets[0], buckets[1]}; with `first`,
    only keys whose first bucket (where an insert looks first) is that one"""
    want = frozenset(buckets)
    assert len(want) == 2 or nb == 1
    out, start, chunk = [], 1, 1 << 18
    while len(out) < n:
        w0, h = _candidates(seed, length, start, chunk, fill)
        tag, b1 = key_tag(h), key_bucket(h, nb)
        b2 = alt_bucket(b1, tag, nb)
        lo, hi = np.minimum(b1, b2), np.maximum(b1, b2)
        ok = (lo == min(want)) & (hi == max(want))
        if first is not None:
            ok &= b1 == first
        hit = np.nonzero(ok)[0]
        out.extend(_key(w0[i], length, fill) for i in hit[: n - len(out)])
        start += chunk
        assert start < (1 << 26), "no keys on this bucket pair"
    return tuple(out)


def key_in_bucket(seed: int, nb: int, bucket: int, length: int, fill: int = 0x69) -> bytes:
    """a key of `length` bytes whose first bucket is `bucket`"""
    w0, h = _candidates(seed, length, 1, 1 << 16, fill)
    return _key(w0[int(np.nonzero(key_bucket(h, nb) == bucket)[0][0])], length, fill)


@functools.lru_cache(maxsize=None)
def full_pair(seed: int, nb: int, n: int, length: int = 8, fill: int = 0x5A):
    """(pair, keys): `n` keys of `length` bytes on the bucket pair most candidates share"""
    w0, h = _candidates(seed, length, 1, 1 << 18, fill)
    tag, b1 = key_tag(h), key_bucket(h, nb)
    b2 = alt_bucket(b1, tag, nb)
    code = np.minimum(b1, b2).astype(np.int64) * nb + np.maximum(b1, b2)
    best = int(np.bincount(code).argmax())
    p = (best // nb, best % nb)
    return p, keys_on_pair(seed, nb, p, n, length, fill)


@functools.lru_cache(maxsize=None)
def twins(seed: int, nb: int, length: int = 8, count: int = 4, fill: int = 0x3C):
    """`count` fingerprint twins of `length` bytes: pairs (a, b) with the same tag whose bucket pairs
    overlap (for two buckets or more, an alternate bucket that is a function of the tag means the
    overlap is the same pair)"""
    out, start, chunk = [], 1, 1 << 22
    while len(out) < count:
        w0, h = _candidates(seed, length, start, chunk, fill)
        tag, b1 = key_tag(h), key_bucket(h, nb)
        order = np.argsort(tag, kind="stable")
        st = tag[order]
        same = np.nonzero(st[1:] == st[:-1])[0]
        for j in same:
            i, k = int(order[j]), int(order[j + 1])
            d = int(alt_bucket(0, tag[i], nb))
            if b1[k] == b1[i] or b1[k] == (b1[i] ^ d):
                out.append((_key(w0[i], length, fill), _key(w0[k], length, fill)))
                if len(out) == count:
                    break
        start += chunk
        assert start < (1 << 27), "no fingerprint twins"
    return tuple(out)


# Keys k (7 bytes) such that k and k + b"\0" are fingerprint twins in a 128-bucket table: their
# 64-bit words are identical, so only the lengths tell them apart.  A twin of this kind has a
# per-key chance of about 2^-37; they were found by a brute-force search over the first word (seconds
# to minutes of compiled code on eight cores) and are checked against the model by test_key_hash_model.py.
LENGTH_TWINS = {
    DEFAULT_SEED: 0x0050E933A090DE6A,
    0xF00DFACE12345679: 0x009B6E878D244F94,
}


def length_twin(seed: int) -> bytes:
    return LENGTH_TWINS[seed].to_bytes(8, "little")[:7]


def is_twin(a: bytes, b: bytes, seed: int, nb: int) -> bool:
    ta, a1, a2 = place(a, seed, nb)
    tb, b1, b2 = place(b, seed, nb)
    return a != b and ta == tb and bool({a1, a2} & {b1, b2})
