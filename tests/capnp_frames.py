"""Hand-laid Cap'n Proto frames of the cdn-proto messages the broker reads, and a mutator that knows
where their decoder-trusted fields are.

The oracle's encoder (``oracle.serialize``) emits one layout: the root struct, the variant struct and
the byte lists in that order behind near pointers, one single far pointer per list that leaves the
1024-word first segment.  A peer may send any layout the encoding spec allows, and a broken or hostile
one sends layouts it does not.  ``frame(Spec(...))`` lays a message out explicitly:

- any number of segments (empty ones appended with ``extra_segs``), a table that claims another count,
  odd and even counts (the table is padded to a word; ``table_pad`` fills the padding);
- every object reached by a near pointer (forward, or backward = negative offset), a single far
  pointer (landing pad at the first or the last word of the object's segment) or a double far pointer
  (two-word pad in a segment of its own; ``tag_off`` goes into the tag word's offset, which readers
  ignore) — separately for the root struct, the Direct/Broadcast struct and each byte list;
- data and pointer sections larger than the schema's (``dw``/``pw`` of the root, ``vd``/``vp`` of the
  variant; extra data words hold junk, extra pointers point nowhere and must never be followed) or
  smaller (absent fields read as empty);
- null pointers for the variant struct and each list, any list element size, a list that claims one
  word past the end of its segment (``over``), bytes after the last segment (``tail``).

Two decisions of the engine's parser (and the oracle's), both listed in DESIGN.md §1, are what the
families below assume: a byte list — Data, and the List(UInt8) topic lists — must have element size
BYTE, where capnp-rust would also read a topic list of wider elements through their low bytes; and the
authentication variants (tags 0–2) are accepted without reading their pointer, which the builder leaves
null for them.

``expected(spec)`` is what a correct decoder reads from ``frame(spec)`` — ``(kind, field 0, field 1)``
with field 0 = recipient / topic list / sync blob — or None when the frame must be rejected.
``tests/test_capnp_frames.py`` pins both against the oracle's decoder and the engine's parser.
"""
from __future__ import annotations

import dataclasses
import random
import struct
from typing import Dict, List, Optional, Tuple

STRUCT, LIST, FAR = 0, 1, 2
BYTE = 2                                   # element size code of Data / List(UInt8)
DIRECT, BROADCAST, SUBSCRIBE, UNSUBSCRIBE, USER_SYNC, TOPIC_SYNC = 3, 4, 5, 6, 7, 8
M32 = (1 << 32) - 1
JUNK_DATA = 0x5A5A_0000_C3C3_0000           # data words of fields the schema does not have
JUNK_PTR = (0x7FFF << 32) | 2               # a far pointer to a segment no frame has: never followed


def struct_tag(dw: int, pw: int) -> int:
    return STRUCT | (dw << 32) | (pw << 48)


def list_tag(esize: int, count: int) -> int:
    return LIST | ((esize | (count << 3)) << 32)


def near_ptr(tag: int, off: int) -> int:
    """`tag` (a pointer with a zero offset) pointing `off` words past the word after the pointer"""
    return (tag & ~M32) | (tag & 3) | ((off << 2) & M32)


def far_ptr(pad: int, seg: int, double: bool = False) -> int:
    return FAR | (4 if double else 0) | ((pad << 3) & M32) | (seg << 32)


@dataclasses.dataclass
class Spec:
    kind: int
    f0: bytes = b""                        # Direct.recipient / Broadcast.topics / Subscribe topics / sync blob
    f1: bytes = b""                        # Direct.message / Broadcast.message
    root: str = "near"                     # how the root struct is reached: near / far / dfar
    var: str = "near"                      # the Direct / Broadcast struct: near / far / dfar / null
    lists: Tuple[str, str] = ("near", "near")   # field 0 / field 1: near / far / dfar / null
    backward: bool = False                 # objects before the pointers that name them (negative offsets)
    pad_last: bool = False                 # landing pads at the end of their segment, not the start
    dw: int = 1
    pw: int = 1
    vd: int = 0
    vp: int = 2
    esize: Tuple[int, int] = (BYTE, BYTE)
    tag: Optional[int] = None              # the union tag word (default: kind); its upper 48 bits are other fields
    tag_off: int = 0
    extra_segs: int = 0
    claim: Optional[int] = None            # segment count the table claims (default: the real one)
    table_pad: int = 0
    tail: bytes = b""
    over: Optional[int] = None             # field whose list claims one word past its segment's end

    def replace(self, **kw) -> "Spec":
        return dataclasses.replace(self, **kw)


class Layout:
    """segments of 64-bit words; `marks` = (what, seg, word) of every field a decoder trusts"""

    def __init__(self):
        self.segs: List[List[int]] = []
        self.marks: List[Tuple[str, int, int]] = []

    def segment(self) -> int:
        self.segs.append([])
        return len(self.segs) - 1

    def alloc(self, seg: int, n: int, fill: int = 0) -> int:
        at = len(self.segs[seg])
        self.segs[seg].extend([fill] * n)
        return at

    def point(self, src, obj, tag: int, how: str, pad=None, tag_off: int = 0) -> None:
        """store at `src` = (seg, word) a pointer to the object at `obj` described by `tag`: near (same
        segment), far (single far, landing pad word `pad` in the object's segment) or dfar (double far,
        two-word pad at `pad`)"""
        (ss, sw), (osg, ow) = src, obj
        if how == "near":
            assert ss == osg
            self.segs[ss][sw] = near_ptr(tag, ow - sw - 1)
            self.marks.append(("ptr", ss, sw))
        elif how == "far":
            ps, pw = pad
            assert ps == osg
            self.segs[ps][pw] = near_ptr(tag, ow - pw - 1)
            self.segs[ss][sw] = far_ptr(pw, ps)
            self.marks += [("far", ss, sw), ("ptr", ps, pw)]
        else:
            ps, pw = pad
            self.segs[ps][pw] = far_ptr(ow, osg)
            self.segs[ps][pw + 1] = near_ptr(tag, tag_off)
            self.segs[ss][sw] = far_ptr(pw, ps, double=True)
            self.marks += [("far", ss, sw), ("far", ps, pw), ("ptr", ps, pw + 1)]

    def table_bytes(self, n: Optional[int] = None) -> int:
        n = len(self.segs) if n is None else n
        return (4 + 4 * n + 7) & ~7

    def offset(self, seg: int, word: int) -> int:
        """byte offset of a word in the encoded frame"""
        return self.table_bytes() + 8 * (sum(len(s) for s in self.segs[:seg]) + word)

    def encode(self, claim: Optional[int] = None, table_pad: int = 0, tail: bytes = b"") -> bytes:
        n = len(self.segs)
        head = struct.pack("<I", (n if claim is None else claim) - 1) + struct.pack(f"<{n}I", *(len(s) for s in self.segs))
        if n % 2 == 0:
            head += struct.pack("<I", table_pad)
        return head + b"".join(struct.pack(f"<{len(s)}Q", *s) for s in self.segs) + tail


def _words(n: int) -> int:
    return (n + 7) // 8


def build(spec: Spec) -> Tuple[bytes, Layout]:
    """the frame of `spec` and its layout (for the mutator)"""
    L = Layout()
    L.segment()
    L.alloc(0, 1)                                          # root pointer
    # objects: name -> [words, parent name or None, pointer index in the parent, how reached]
    objs: Dict[str, list] = {"R": [spec.dw + spec.pw, None, 0, spec.root]}
    fields = {}
    if spec.kind in (DIRECT, BROADCAST):
        if spec.pw >= 1 and spec.var != "null":
            objs["V"] = [spec.vd + spec.vp, "R", spec.dw, spec.var]
            for i, data in enumerate((spec.f0, spec.f1)):
                if spec.vp > i and spec.lists[i] != "null":
                    objs[f"L{i}"] = [_words(len(data)), "V", spec.vd + i, spec.lists[i]]
                    fields[f"L{i}"] = (data, spec.esize[i], i)
    elif spec.kind in (SUBSCRIBE, UNSUBSCRIBE, USER_SYNC, TOPIC_SYNC):
        if spec.pw >= 1 and spec.lists[0] != "null":
            objs["L0"] = [_words(len(spec.f0)), "R", spec.dw, spec.lists[0]]
            fields["L0"] = (spec.f0, spec.esize[0], 0)
    # segments: a near object lives in its parent's segment, a far one in a new segment
    seg_of: Dict[str, int] = {}
    for name in ("R", "V", "L0", "L1"):
        if name in objs:
            parent, how = objs[name][1], objs[name][3]
            seg_of[name] = (seg_of[parent] if parent else 0) if how == "near" else L.segment()
    pads: Dict[str, Tuple[int, int]] = {}
    order = ("L1", "L0", "V", "R") if spec.backward else ("R", "V", "L0", "L1")
    at: Dict[str, Tuple[int, int]] = {}
    for s in range(len(L.segs)):
        here = [n for n in order if n in objs and seg_of[n] == s]
        far_here = [n for n in here if objs[n][3] == "far"]
        if not spec.pad_last:
            for n in far_here:
                pads[n] = (s, L.alloc(s, 1))
        for n in here:
            at[n] = (s, L.alloc(s, objs[n][0]))
        if spec.pad_last:
            for n in far_here:
                pads[n] = (s, L.alloc(s, 1))
    for n in order:                                        # double-far pads: a segment each
        if n in objs and objs[n][3] == "dfar":
            s = L.segment()
            if spec.pad_last:
                L.alloc(s, 1, JUNK_DATA)
            pads[n] = (s, L.alloc(s, 2))
            if not spec.pad_last:
                L.alloc(s, 1, JUNK_DATA)
    for _ in range(spec.extra_segs):
        L.segment()
    # contents
    rs, rw = at["R"]
    if spec.dw:
        L.segs[rs][rw] = spec.kind if spec.tag is None else spec.tag
        L.marks.append(("tag", rs, rw))
        for k in range(1, spec.dw):
            L.segs[rs][rw + k] = JUNK_DATA
    for k in range(1, spec.pw):                            # pointers beyond the schema's one
        L.segs[rs][rw + spec.dw + k] = JUNK_PTR
    if "V" in at:
        vs, vw = at["V"]
        for k in range(spec.vd):
            L.segs[vs][vw + k] = JUNK_DATA
        for k in range(2, spec.vp):
            L.segs[vs][vw + spec.vd + k] = JUNK_PTR
    for name, (data, esize, i) in fields.items():
        s, w = at[name]
        padded = data + bytes(-len(data) % 8)
        L.segs[s][w:w + len(padded) // 8] = list(struct.unpack(f"<{len(padded) // 8}Q", padded))
    # pointers
    for name in ("R", "V", "L0", "L1"):
        if name not in objs:
            continue
        words, parent, idx, how = objs[name]
        src = (0, 0) if parent is None else (at[parent][0], at[parent][1] + idx)
        if name == "R":
            tag = struct_tag(spec.dw, spec.pw)
        elif name == "V":
            tag = struct_tag(spec.vd, spec.vp)
        else:
            data, esize, i = fields[name]
            count = len(data) if spec.over != i else words * 8 + 1
            tag = list_tag(esize, count)
        L.point(src, at[name], tag, how, pads.get(name), spec.tag_off)
    return L.encode(spec.claim, spec.table_pad, spec.tail), L


def frame(spec: Spec) -> bytes:
    return build(spec)[0]


def expected(spec: Spec):
    """(kind, field 0, field 1) a correct decoder reads from frame(spec), or None = malformed"""
    assert spec.claim is None or spec.claim >= 512, "a table that claims fewer segments than 512 is not modelled"
    tag = (spec.kind if spec.tag is None else spec.tag) & 0xFFFF if spec.dw else 0
    if tag > 8 or spec.claim is not None or len(build(spec)[1].segs) >= 512:   # capnp-rust: "Too many segments"
        return None
    if tag in (DIRECT, BROADCAST):
        if spec.pw < 1 or spec.var == "null":
            return tag, b"", b""
        out = []
        for i, data in enumerate((spec.f0, spec.f1)):
            if spec.vp <= i or spec.lists[i] == "null":
                out.append(b"")
                continue
            if spec.esize[i] != BYTE or spec.over == i:
                return None
            out.append(data)
        return tag, out[0], out[1]
    if tag in (SUBSCRIBE, UNSUBSCRIBE, USER_SYNC, TOPIC_SYNC):
        if spec.pw < 1 or spec.lists[0] == "null":
            return tag, b"", b""
        if spec.esize[0] != BYTE or spec.over == 0:
            return None
        return tag, spec.f0, b""
    return tag, b"", b""


# ------------------------------------------------------------------------------------- families
# Layout families a peer may send: every one is a valid frame of any kind and field contents.
FAMILIES: Dict[str, dict] = {
    "near": {},
    "backward": dict(backward=True),
    "root-far": dict(root="far"),
    "root-far-pad-last": dict(root="far", pad_last=True),
    "root-dfar": dict(root="dfar", tag_off=3),
    "var-far": dict(var="far"),
    "var-far-pad-last": dict(var="far", pad_last=True, backward=True),
    "var-dfar": dict(var="dfar", tag_off=-2),
    "var-null": dict(var="null"),
    "f0-far": dict(lists=("far", "near")),
    "f0-dfar": dict(lists=("dfar", "near"), tag_off=7),
    "f0-null": dict(lists=("null", "near")),
    "f1-far": dict(lists=("near", "far")),
    "f1-dfar": dict(lists=("near", "dfar"), pad_last=True, tag_off=1),
    "f1-null": dict(lists=("near", "null")),
    "lists-far-pad-last": dict(lists=("far", "far"), pad_last=True),
    "all-dfar": dict(root="dfar", var="dfar", lists=("dfar", "dfar"), tag_off=5),
    "all-dfar-pad-last": dict(root="dfar", var="dfar", lists=("dfar", "dfar"), pad_last=True, tag_off=-9, backward=True),
    "mixed-far": dict(root="far", var="dfar", lists=("far", "dfar"), tag_off=2),
    "newer-root": dict(dw=3, pw=2, tag_off=0),
    "newer-var": dict(vd=2, vp=4),
    "newer-both-far": dict(dw=2, pw=3, vd=1, vp=3, var="far", lists=("dfar", "far"), tag_off=4),
    "older-var": dict(vp=1),
    "empty-var": dict(vp=0, vd=1),
    "root-no-pointers": dict(pw=0),
    "root-no-data": dict(dw=0),
    "tag-upper-bits": dict(tag=None),
    "segs-odd": dict(extra_segs=2, table_pad=0),
    "segs-even-pad": dict(extra_segs=1, table_pad=0xDEADBEEF),
    "segs-511": dict(extra_segs=508, lists=("far", "far")),      # 1 + 2 + 508 segments
    "trailing-bytes": dict(tail=b"\x01" * 8 + b"tail"),
    "exact-segment-end": dict(lists=("far", "far")),
}

# Frames that must be rejected.
MALFORMED: Dict[str, dict] = {
    "segs-512": dict(extra_segs=511),
    "table-claims-512": dict(claim=512),
    "f0-over-segment-end": dict(lists=("far", "near"), over=0),
    "f1-over-segment-end": dict(over=1, extra_segs=1),
    "f1-far-over": dict(lists=("near", "far"), over=1),
    "f0-over-into-next-segment": dict(lists=("far", "far"), over=0),   # the word past it is segment data
    "tag-9": dict(tag=9),
    "tag-ffff": dict(tag=0xFFFF),
    **{f"f0-esize-{k}": dict(esize=(k, BYTE)) for k in range(8) if k != BYTE},
    **{f"f1-esize-{k}": dict(esize=(BYTE, k)) for k in range(8) if k != BYTE},
}


def family_spec(name: str, kind: int, f0: bytes, f1: bytes) -> Spec:
    kw = dict(FAMILIES[name] if name in FAMILIES else MALFORMED[name])
    if name == "tag-upper-bits":
        kw["tag"] = kind | (0xBEEF << 16) | (0x1234 << 48)
    return Spec(kind, f0, f1, **kw)


def applies(name: str, kind: int) -> bool:
    """a family that only changes what `kind` does not have is left out for it"""
    kw = FAMILIES[name] if name in FAMILIES else MALFORMED[name]
    variant = kind in (DIRECT, BROADCAST)
    if not variant and (kw.get("var") not in (None, "near") or "vd" in kw or "vp" in kw or
                        (kw.get("lists", ("near", "near"))[1] != "near") or kw.get("over") == 1 or
                        kw.get("esize", (BYTE, BYTE))[1] != BYTE):
        return False
    if kind < DIRECT and ("lists" in kw or "esize" in kw or "over" in kw):
        return False
    return True


KINDS = (DIRECT, BROADCAST, SUBSCRIBE, UNSUBSCRIBE, USER_SYNC, TOPIC_SYNC, 0)
# message sizes on both sides of the 1024-word segment the reference's encoder starts with
PAYLOADS = (0, 9, 8 * 1024 - 64, 8 * 1024 + 8)


def field_sizes(max_key_len: int) -> Tuple[int, ...]:
    return (0, 1, 7, 8, 9, max_key_len - 1, max_key_len, max_key_len + 1)


def key_of(n: int) -> bytes:
    """the recipient key of length n the corpus sends Direct frames to"""
    return bytes((7 * i + n) & 0xFF for i in range(n))


def field0(kind: int, n: int, n_topics: int = 5) -> bytes:
    if kind == DIRECT:
        return key_of(n)
    if kind in (BROADCAST, SUBSCRIBE, UNSUBSCRIBE):
        return bytes((i * 3 + n) % n_topics for i in range(n))
    return bytes((i * 11 + 1) & 0xFF for i in range(n))


def corpus(max_key_len: int, families=None, kinds=KINDS):
    """(name, spec) of every layout family (valid and malformed) × kind × field size; field 1 sizes
    cycle through PAYLOADS"""
    out = []
    for fam in families or list(FAMILIES) + list(MALFORMED):
        for kind in kinds:
            if not applies(fam, kind):
                continue
            for j, n in enumerate(field_sizes(max_key_len)):
                f1 = bytes([(j * 37 + 5) & 0xFF]) * PAYLOADS[j % len(PAYLOADS)] if kind in (DIRECT, BROADCAST) else b""
                out.append((f"{fam}/{kind}/{n}", family_spec(fam, kind, field0(kind, n), f1)))
    return out


# ------------------------------------------------------------------------------------- mutation
def mutate(rng: random.Random, raw: bytes, layout: Layout) -> bytes:
    """change one or two fields a decoder trusts: the segment count or a size in the table, a pointer's
    kind bits / offset / far and double-far bits / target segment, a list's element size or count, or
    the union tag (8, 9, 0xFFFF)"""
    b = bytearray(raw)
    n = len(layout.segs)
    for _ in range(rng.randrange(1, 3)):
        r = rng.random()
        if r < 0.15:                                          # segment table
            i = rng.randrange(n + 1)
            old = struct.unpack_from("<I", b, 4 * i)[0]
            new = rng.choice([old + 1, max(old - 1, 0), 0, old + rng.randrange(2, 64), 511, 512, 0xFFFFFFFF])
            struct.pack_into("<I", b, 4 * i, new & M32)
            continue
        marks = layout.marks
        what, s, w = marks[rng.randrange(len(marks))]
        off = layout.offset(s, w)
        v = struct.unpack_from("<Q", b, off)[0]
        if what == "tag":
            v = (v & ~0xFFFF) | rng.choice([8, 9, 0xFFFF, 3, 4, 5])
        elif what == "far":
            c = rng.randrange(4)
            if c == 0:
                v ^= 4                                        # single <-> double far
            elif c == 1:
                v = (v & M32) | (rng.choice([0, 1, 2, n - 1, n, n + 1, 0xFFFF]) << 32)   # target segment
            elif c == 2:                                      # landing pad position
                pad = ((v & M32) >> 3) + rng.choice([-2, -1, 1, 2, 1 << 20])
                v = (v & ~M32) | (v & 7) | ((pad << 3) & M32)
            else:
                v = (v & ~3) | rng.choice([0, 1, 3])          # no longer a far pointer
        else:
            c = rng.randrange(4)
            if c == 0:
                v = (v & ~3) | rng.choice([0, 1, 2, 3])       # pointer kind bits
            elif c == 1:
                o = ((v & M32) >> 2) - ((v & M32) >> 31 << 30)
                o += rng.choice([-(1 << 29), -3, -1, 1, 2, 9, 1 << 20])
                v = (v & ~M32) | (v & 3) | ((o << 2) & M32)
            elif c == 2 and (v & 3) == LIST:
                v = (v & ~(7 << 32)) | (rng.randrange(8) << 32)    # element size
            else:
                hi = v >> 32
                if (v & 3) == LIST:
                    cnt = (hi >> 3) + rng.choice([-9, -8, -1, 1, 7, 8, 9, 1 << 20, (1 << 29) - 1 - (hi >> 3)])
                    hi = (hi & 7) | ((max(cnt, 0) << 3) & M32)
                else:
                    hi = hi ^ (rng.choice([1, 2, 0xFFFF]) << rng.choice([0, 16]))   # data / pointer words
                v = (v & M32) | (hi << 32)
        struct.pack_into("<Q", b, off, v & ((1 << 64) - 1))
    return bytes(b)
