"""The device's direct-key lookup (kernels.cu direct_lookup_body: k_direct_lookup and the fused
k_ctrl_small) at the inputs where a partial-key cuckoo lookup goes wrong: fingerprint twins (same tag,
overlapping bucket pair) that only the full-key compare and the length check tell apart, every key
length around the word and lane boundaries, non-zero bytes after a key read in place, full bucket
pairs, entries relocated to their alternate bucket, one- and two-bucket tables, a key slot reused
while the batch that named its old key is in flight, remote routes, and hot recipients.  The
collisions come from the hash model in keyhash.py (pinned on the CPU by test_key_hash_model.py).

Every batch is compared with the oracle's plain hash map bit for bit, n_direct_dropped with the
number of directs the oracle delivered nowhere, and debug_route with the oracle's route of every key
a test touched.  One difference is deliberate: the engine refuses a key whose bucket pair is full
(PCDN_ENOSPC), where the reference's map never refuses; such a key is never given to the oracle.
"""
import random

import pytest

from gpu_world import PCDN_ENOSPC, World
import keyhash as kh
from kconst import K
from oracle import oracle as orc

pytestmark = pytest.mark.gpu

SEEDS = [0, 0xF00DFACE12345679]          # 0: the built-in seed
SEED_IDS = ["builtin-seed", "top-bit-seed"]
MAX_KEYS = 256                           # 128 buckets
SENDER = b"sender"                       # receive paths: the user a frame comes from (never registered)

# control path / ingress path.  fused: small engine, <= 256 messages (k_ctrl_small); staged:
# FLAG_STAGED_SPANS (regular kernels); big: every batch padded past 256 messages; shards: three
# connection shards on GPU 0 (conn_base != 0).  handle: key staged beside the frame; host-parse: the
# key read in place inside the frame; device-parse: k_parse sets the key offset; submit-device: a
# device-resident batch with its keys behind the frames.
PATHS = ["fused/handle", "fused/host-parse", "fused/device-parse", "fused/submit-device",
         "staged/handle", "staged/device-parse", "big/handle", "big/host-parse",
         "shards/handle", "shards/device-parse", "shards/submit-device"]
BIG_PAD = 300


class Lookup:
    """a World (engine + oracle) whose directs all go through one control / ingress path"""

    def __init__(self, pcdn, path, seed, max_keys=MAX_KEYS, max_key_len=64, **cfg):
        ctrl, self.ingress = path.split("/")
        flags = 0
        kw = dict(max_conns=256, max_topics=16, max_keys=max_keys, max_key_len=max_key_len, hash_seed=seed,
                  ring_bytes_per_conn=1 << 16, max_batch_msgs=4096, max_batch_bcast=16, max_batch_bytes=4 << 20,
                  max_batch_deliveries=1 << 14)
        if ctrl == "staged":
            flags |= pcdn.FLAG_STAGED_SPANS
        if ctrl == "shards":
            kw.update(devices=[0, 0, 0], ingest=pcdn.INGEST_HOST)
        if self.ingress == "device-parse":
            flags |= pcdn.FLAG_DEVICE_PARSE
        kw.update(cfg)
        self.pcdn = pcdn
        self.w = World(pcdn, flags=flags, **kw)
        self.pad = ctrl == "big"
        self.seed, self.nb, self.max_key_len = kh.engine_seed(seed), kh.n_buckets(max_keys), max_key_len
        self.touched = set()
        self.n = 0
        self.keep = []                   # device-resident batches stay allocated until they are drained

    # ---- state (engine and oracle) ----
    def add(self, key):
        self.touched.add(key)
        return self.w.add_user(key, [])

    def refuse(self, key):
        """the engine refuses `key` for lack of a slot; the oracle never sees it"""
        self.touched.add(key)
        with pytest.raises(self.pcdn.PcdnError) as ei:
            self.w.e.add_user(key, [])
        assert ei.value.code == PCDN_ENOSPC

    def remove(self, key):
        self.touched.add(key)
        self.w.both("remove_user", key)

    # ---- data ----
    def frame(self, rcpt, dirty=False):
        """a direct frame to `rcpt`; dirty: the recipient's Data padding up to the next word is non-zero"""
        self.n += 1
        raw = orc.direct_frame(rcpt, b"m%d:" % self.n + rcpt[:3])
        if dirty:
            _, _, (off, ln) = self.pcdn.parse_frame(raw)
            end = (off + ln + 7) // 8 * 8
            b = bytearray(raw)
            b[off + ln:end] = bytes(0xA5 ^ i for i in range(end - off - ln))
            raw = bytes(b)
            assert orc.deserialize(raw)[1] == rcpt and self.pcdn.parse_frame(raw)[2] == (off, ln)
        return raw

    def send(self, rcpts, origin=0, dirty=False):
        """one batch of directs (broker origin = to_user_only); rcpts may carry their own origin as (key, origin)"""
        msgs = [(r, origin) if isinstance(r, bytes) else r for r in rcpts]
        if self.pad:
            msgs += [(b"pad-%d" % i, 0) for i in range(BIG_PAD)]
        msgs = [(k, o, self.frame(k, dirty)) for k, o in msgs]
        self.touched.update(k for k, _, _ in msgs)
        if self.ingress == "handle":
            for k, o, raw in msgs:
                self.w.direct(k, raw, bool(o))
        elif self.ingress in ("host-parse", "device-parse"):
            want = [self.w.o.broker_receive(raw) if o else self.w.o.user_receive(SENDER, raw) for k, o, raw in msgs]
            assert self.w.e.receive_frames([(SENDER, o, raw) for k, o, raw in msgs]) == want == [0] * len(msgs)
        else:
            self._submit_device(msgs)
        return len(msgs)

    def _submit_device(self, msgs):
        import torch

        arena, kinds, flags, slot, aoff, alen = bytearray(), [], [], [], [], []
        for k, o, raw in msgs:
            self.w.o.handle_direct_message(k, raw, bool(o))
            slot.append(len(arena) // 16)
            arena += bytes(4) + raw + bytes((-(4 + len(raw))) % 16)
            aoff.append(len(arena))
            alen.append(len(k))
            # the key at a 4-byte aligned offset, garbage behind it up to the next 16 bytes and beyond
            arena += k + bytes((0x5A + i) & 255 or 1 for i in range((-len(k)) % 16 + 16))
            kinds.append(3)
            flags.append(1 if o else 0)
        dev = torch.device("cuda", self.w.e.shard_info(0).device)
        t8 = lambda a: torch.tensor(list(a), dtype=torch.uint8, device=dev)
        t32 = lambda a: torch.tensor(list(a), dtype=torch.int32, device=dev)
        a = [t8(arena + bytes(64)), t8(kinds), t8(flags), t32(slot), t32([len(r) for _, _, r in msgs]),
             t32(aoff), t32(alen), torch.zeros(1, dtype=torch.int16, device=dev), torch.zeros(1, dtype=torch.int32, device=dev)]
        self.keep.append(a)
        torch.cuda.synchronize(dev)
        db = self.pcdn.DeviceBatch(len(msgs), 0, a[0].data_ptr(), len(arena), a[1].data_ptr(), a[2].data_ptr(),
                                   a[3].data_ptr(), a[4].data_ptr(), a[5].data_ptr(), a[6].data_ptr(), a[7].data_ptr(), 0,
                                   a[8].data_ptr())
        self.w.e.submit_device(db)

    def check(self, n_msgs):
        """every outstanding batch against the oracle; they held n_msgs directs in all, and the ones the
        oracle delivered nowhere are the ones the engine counted as dropped"""
        e = self.w.e
        e.flush()
        got, seen, dropped = {}, 0, 0
        while True:
            b = e.next_batch()
            if not b:
                break
            res = e.poll(b)
            assert res.status == 0 and res.n_overflow == 0 and res.n_msg_errors == 0
            seen += res.n_msgs
            dropped += res.n_direct_dropped
            for conn, fr in e.collect_frames(res).items():
                got.setdefault(conn, []).extend(fr)
            e.last_result = res
            e.release_batch(b)
        self.keep.clear()
        want = self.w.expect()
        delivered = self.w.compare(e, got, want)
        assert seen == n_msgs
        assert dropped == n_msgs - delivered
        self.check_routes()
        return delivered

    def check_routes(self):
        for k in sorted(self.touched):
            kind, conn = self.w.e.debug_route(k)
            okind, oconn = self.w.o.route(k)
            assert kind == okind, k
            assert (conn == -1) == (oconn == -1), k
            if conn != -1:
                assert self.w.map[conn] == oconn, k

    def model_twins(self, length, count):
        return kh.twins(self.seed, self.nb, length, count)

    def close(self):
        self.w.e.close()


@pytest.fixture(params=SEEDS, ids=SEED_IDS)
def seed(request):
    return request.param


def _mixed(groups):
    """interleave the outcome lists so that every four consecutive messages (the four groups of one
    warp) mix them: group k of the warp takes list (j + k) % len(groups) for warp j"""
    n = max(len(g) for g in groups)
    out = []
    for j in range(n):
        for k in range(4):
            g = groups[(j + k) % len(groups)]
            out.append(g[(j * 4 + k) % len(g)])
    return out


# ------------------------------------------------------------------------------ 1. fingerprint twins
@pytest.mark.parametrize("path", PATHS)
def test_fingerprint_twins(pcdn, path, seed):
    """Twins registered in both orders (so the wrong twin is sometimes the first candidate in slot
    order), a twin whose other half is not registered (dropped and counted once), and the twins k /
    k + b"\\0" whose words are identical; the four groups of every warp mix twin hits, twin misses,
    plain hits and unknown keys, so they take different numbers of passes through the candidate loop."""
    L = Lookup(pcdn, path, seed)
    tw = list(L.model_twins(8, 3)) + list(L.model_twins(13, 1))
    lt = kh.length_twin(L.seed)
    both = [tw[0], tw[1][::-1], tw[3], (lt + b"\0", lt)]
    for a, b in both:
        L.add(a)
        L.add(b)
    half, missing = tw[2]
    L.add(half)
    plain = [b"plain-key-%d" % i for i in range(6)]
    for k in plain:
        L.add(k)
    hits = [k for p in both for k in p] + [half]
    unknown = [b"unknown-%d" % i for i in range(5)] + [b"", b"plain-key-"]
    n = L.send(_mixed([hits, [missing], plain, unknown]))
    assert L.check(n) > 0
    # the other registration order, and the missing twin now registered while its partner is not
    for a, b in both:
        L.remove(a)
        L.remove(b)
    L.remove(half)
    for a, b in both:
        L.add(b)
        L.add(a)
    L.add(missing)
    n = L.send(_mixed([hits, [missing, half], plain, unknown]))
    L.check(n)
    L.close()


# ------------------------------------------------------------------------------ 2. every key length
LENGTHS = [0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 15, 16, 17, 63, 64, 65, 127, 128, 129, 255, 256, 257]


@pytest.mark.parametrize("max_key_len", [20, 300])
@pytest.mark.parametrize("path", PATHS)
def test_every_key_length(pcdn, path, seed, max_key_len):
    """Keys of every length around the 4- and 8-byte words and the eight hashing lanes (0..9, 15..17,
    63..65, 127..129, 255..257, limit - 1, limit) that are prefixes of one another, keys that differ
    from them only in their last byte (registered for every other length, unknown for the rest), and a
    recipient one byte over the limit, whose registered prefixes include the empty key.
    max_key_len 20 makes the key stride (32) larger than the limit."""
    L = Lookup(pcdn, path, seed, max_key_len=max_key_len, max_keys=512)
    rng = random.Random(max_key_len)
    root = bytes(rng.randrange(1, 256) for _ in range(max_key_len + 1))
    lens = sorted({n for n in LENGTHS if n <= max_key_len} | {max_key_len - 1, max_key_len})
    chain = [root[:n] for n in lens]
    last = [k[:-1] + bytes([k[-1] ^ 0x01]) for k in chain if k]
    for k in chain:
        L.add(k)                      # the engine takes the empty key as the reference's map does
    for i, k in enumerate(last):
        if i % 2 == 0:
            L.add(k)
    over = root[:max_key_len + 1]
    rcpts = chain + last + [over, over[:-1] + b"\xff", root[:max_key_len] + b"\0"]
    n = L.send(_mixed([rcpts[i::3] for i in range(3)]))
    L.check(n)
    L.close()


# ------------------------------------------------------------------------------ 3. non-zero padding
@pytest.mark.parametrize("path", ["fused/host-parse", "fused/device-parse", "staged/device-parse",
                                  "big/host-parse", "shards/device-parse", "fused/submit-device"])
def test_nonzero_bytes_after_the_key(pcdn, path, seed):
    """Direct frames whose recipient Data padding (up to the next word) is non-zero, which the oracle
    accepts: the key is read in place (host parse) or where k_parse found it (device parse), so only
    the tail mask keeps those bytes out of the hash and the compare.  A device-resident batch has
    garbage behind every key (submit-device)."""
    L = Lookup(pcdn, path, seed)
    rng = random.Random(7)
    keys = [bytes(rng.randrange(256) for _ in range(n)) for n in (1, 2, 3, 5, 6, 7, 9, 10, 11, 13, 14, 15, 21, 33)]
    lt = kh.length_twin(L.seed)
    tw = L.model_twins(13, 1)[0]
    for k in keys[::2] + [lt, lt + b"\0", tw[0], tw[1]]:
        L.add(k)
    n = L.send(keys + [lt, lt + b"\0", tw[0], tw[1]], dirty=True)
    L.check(n)
    L.close()


# ------------------------------------------------------------------------------ 4. full bucket pairs
@pytest.mark.parametrize("path", PATHS)
def test_full_bucket_pair(pcdn, path, seed):
    """Eight keys fill both buckets of one pair; the ninth add_user walks, fails, and rolls every
    eviction back in the same journal flush.  The next batch still routes all eight on the device.
    Then one of the eight goes and the ninth takes its slot: the removed key's directs are dropped."""
    L = Lookup(pcdn, path, seed)
    p, keys = kh.full_pair(L.seed, L.nb, 9)
    for k in keys[:8]:
        L.add(k)
    L.refuse(keys[8])
    batch = _mixed([list(keys), [b"nobody"]])
    n = L.send(batch)
    assert L.check(n) == sum(k in keys[:8] for k in batch)
    L.remove(keys[3])
    L.add(keys[8])
    n = L.send(batch)
    assert L.check(n) == sum(k in keys and k != keys[3] for k in batch)
    L.close()


# ------------------------------------------------------------------------------ 5. relocation
@pytest.mark.parametrize("path", PATHS)
def test_relocated_entries(pcdn, path, seed):
    """A kick walk: bucket Y holds four keys of pair {X, Y} and bucket Z four keys of pair {Z, W}
    (all in their first bucket); a key of pair {Y, Z} finds both full and evicts one of them to its
    alternate bucket, where only the second half of the probing lanes finds it."""
    L = Lookup(pcdn, path, seed)
    s, nb = L.seed, L.nb
    X, Y, Z, W = 3, 40, 77, 100    # pairs differ in an odd number: the tag is odd, so is its alternate offset
    xy = kh.keys_on_pair(s, nb, (X, Y), 4, 8, 0x5A, Y)
    zw = kh.keys_on_pair(s, nb, (Z, W), 4, 12, 0x5A, Z)
    yz = kh.keys_on_pair(s, nb, (Y, Z), 2, 10, 0x5A)
    for k in xy + zw:
        L.add(k)
    n = L.send(list(xy + zw))
    L.check(n)
    L.add(yz[0])                       # evicts one of the eight
    n = L.send(_mixed([list(xy + zw + yz[:1]), [yz[1]]]))
    L.check(n)
    L.add(yz[1])                       # a second walk
    n = L.send(list(xy + zw + yz))
    L.check(n)
    L.close()


# ------------------------------------------------------------------------------ 6. tiny tables
@pytest.mark.parametrize("max_keys", [1, 2, 3])
@pytest.mark.parametrize("path", ["fused/handle", "fused/device-parse", "staged/handle", "shards/submit-device"])
def test_tiny_tables(pcdn, path, seed, max_keys):
    """max_keys 1 and 2: one bucket, b1 == b2, only the first four lanes probe; 3: two buckets.  The
    table holds twins (same tag) where two keys fit; a key beyond max_keys is refused (the engine's
    capacity, which the reference's map does not have)."""
    L = Lookup(pcdn, path, seed, max_keys=max_keys)
    assert L.nb == (1 if max_keys <= 2 else 2)
    lt = kh.length_twin(L.seed)
    a, b = kh.twins(L.seed, L.nb, 8, 1)[0]
    keys = {1: [a], 2: [a, b], 3: [lt, lt + b"\0", a]}[max_keys]
    for k in keys:
        L.add(k)
    L.refuse(b"one too many")
    rcpts = [a, b, lt, lt + b"\0", b"one too many", b"", b"x"]
    n = L.send(rcpts * 3)
    L.check(n)
    L.remove(keys[0])
    L.add(b if max_keys == 1 else b"late")
    n = L.send(rcpts + [b"late"])
    L.check(n)
    L.close()


# ------------------------------------------------------------------------------ 7. slot reuse in flight
@pytest.mark.parametrize("b_len", [5, 20], ids=["shorter", "longer"])
@pytest.mark.parametrize("path", PATHS)
def test_slot_reuse_while_in_flight(pcdn, path, seed, b_len):
    """A direct to A; remove_user(A); add_user(B), which takes A's key slot and (first bucket equal
    to A's, which A had to itself) A's cuckoo slot; a direct to A and one to B.  Nothing is drained in
    between, so the first batch is in flight while the journal rewrites the slot: it must still reach
    A, the second must drop A and reach B (R12)."""
    L = Lookup(pcdn, path, seed)
    A = b"A-key-twelve"
    _, a1, _ = kh.place(A, L.seed, L.nb)
    B = kh.key_in_bucket(L.seed, L.nb, a1, b_len)
    assert kh.place(B, L.seed, L.nb)[1] == a1
    L.add(A)
    n = L.send([A])
    L.remove(A)
    L.add(B)
    n += L.send([A, B])
    assert L.check(n) == 2
    L.close()


# ------------------------------------------------------------------------------ 8. routes on twins
@pytest.mark.parametrize("path", PATHS)
def test_remote_routes_on_twins(pcdn, path, seed):
    """One twin owned by a peer broker (apply_user_sync), the other a local user: user-origin directs
    to the remote twin are forwarded to the peer, broker-origin (to_user_only) ones are dropped.  Then
    the two swap: the local one moves to the peer and the remote one connects here."""
    L = Lookup(pcdn, path, seed)
    L.w.add_broker("1/1")
    for a, b in (L.model_twins(8, 1)[0], (kh.length_twin(L.seed), kh.length_twin(L.seed) + b"\0")):
        L.add(a)
        L.touched.add(b)
        L.w.both("apply_user_sync", "1/1", [(b, 1, "1/1")])
        rc = [(a, 0), (b, 0), (a, 1), (b, 1), (b, 0), (a, 0), (b"nobody", 0), (b, 1)]
        n = L.send(rc)
        L.check(n)
        L.add(b)
        L.w.both("apply_user_sync", "1/1", [(a, 5, "1/1")])
        n = L.send(rc)
        L.check(n)
    L.close()


# ------------------------------------------------------------------------------ 9. a hot twin
@pytest.mark.parametrize("n_hot", [40, 1100])
@pytest.mark.parametrize("path", ["fused/handle", "fused/device-parse", "staged/handle", "shards/host-parse",
                                  "fused/submit-device"])
def test_hot_twin(pcdn, path, seed, n_hot):
    """More than kHotMin (32) directs to one twin, interleaved with directs to the other, in one batch
    (k_dsort_hot orders them); 1100 + 1100 directs also reach kThinSeparateMin (2048)."""
    assert n_hot > K.kHotMin
    if n_hot > 100:
        assert 2 * n_hot >= K.kThinSeparateMin
    L = Lookup(pcdn, path, seed, ring_bytes_per_conn=1 << 18)
    a, b = L.model_twins(8, 1)[0]
    L.add(a)
    L.add(b)
    rc = [a, b] * n_hot + [a] * 7
    n = L.send(rc)
    assert L.check(n) == n - (BIG_PAD if L.pad else 0)
    L.close()
