#!/usr/bin/env python
"""Generate pcdn-sys/src/lib.rs — the Rust `-sys` binding of include/pcdn_fanout.h — from the header.

    python scripts/gen_pcdn_sys.py            # rewrite pcdn-sys/src/lib.rs
    python scripts/gen_pcdn_sys.py --check    # exit 1 if the committed file differs from the header

There is no Rust toolchain in the build image, so the crate is generated and committed UNCOMPILED;
tests/test_pcdn_sys.py runs the --check mode (header and crate cannot drift) and verifies that every
declared function is exported by libpcdn_fanout.so with the same arity.  The parser understands
exactly the C subset the header uses: #define of integer constants, anonymous enums, typedefs of
scalars, opaque and plain structs, function-pointer typedefs and function prototypes.
"""
import os
import re
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "pcdn_fanout.h")
OUT = os.path.join(ROOT, "pcdn-sys", "src", "lib.rs")

SCALARS = {
    "uint8_t": "u8", "uint16_t": "u16", "uint32_t": "u32", "uint64_t": "u64", "int8_t": "i8", "int16_t": "i16",
    "int32_t": "i32", "int64_t": "i64", "int": "c_int", "double": "f64", "float": "f32", "size_t": "usize", "char": "c_char",
    "void": "c_void",
}
KEYWORDS = {"type", "ref", "in", "match", "move", "loop", "fn", "impl", "box", "self", "struct", "use", "mod"}


def strip_comments(src):
    src = re.sub(r"/\*.*?\*/", " ", src, flags=re.S)
    return re.sub(r"//[^\n]*", " ", src)


def rust_type(ctype, known):
    """'const uint8_t*' -> '*const u8'; 'pcdn_engine**' -> '*mut *mut pcdn_engine'"""
    t = ctype.strip()
    stars = t.count("*")
    t = t.replace("*", " ")
    toks = t.split()
    const = "const" in toks
    toks = [x for x in toks if x not in ("const", "struct", "unsigned")]
    assert len(toks) == 1, ctype
    base = toks[0]
    rbase = SCALARS.get(base, base)
    assert base in SCALARS or base in known, "unknown C type %r" % ctype
    if stars == 0:
        assert rbase != "c_void"
        return rbase
    out = rbase
    for i in range(stars):
        # the innermost pointer carries the const qualifier of the pointee
        out = ("*const " if (const and i == 0) else "*mut ") + out
    return out


def ident(name):
    return name + "_" if name in KEYWORDS else name


def parse_params(params, known):
    params = params.strip()
    if params in ("", "void"):
        return []
    out = []
    for i, p in enumerate(params.split(",")):
        p = p.strip()
        m = re.match(r"^(.*?)([A-Za-z_][A-Za-z_0-9]*)$", p)
        assert m, p
        ctype, name = m.group(1), m.group(2)
        if not ctype.strip() or name in SCALARS or name in known:   # unnamed parameter
            ctype, name = p, "arg%d" % i
        out.append((ident(name), rust_type(ctype, known)))
    return out


def generate():
    raw = open(HEADER).read()
    src = strip_comments(raw)
    body = src[src.index('extern "C" {') + len('extern "C" {'):]
    body = body[:body.rindex("#ifdef __cplusplus")]
    consts, types, structs, fnptrs, funcs = [], [], [], [], []
    known = set()
    for m in re.finditer(r"#define\s+(PCDN_[A-Z_0-9]+)\s+(0x[0-9A-Fa-f]+|\d+)u?\b", src):
        if m.group(1) == "PCDN_FANOUT_H":
            continue
        v = m.group(2)
        consts.append((m.group(1), "u32", v))
    body = re.sub(r"#[^\n]*", " ", body)
    # split into top-level declarations at ';' outside braces
    decls, depth, cur = [], 0, []
    for ch in body:
        if ch == "{":
            depth += 1
        elif ch == "}":
            depth -= 1
        if ch == ";" and depth == 0:
            decls.append("".join(cur).strip())
            cur = []
        else:
            cur.append(ch)
    for d in decls:
        d = " ".join(d.split())
        if not d:
            continue
        m = re.match(r"^enum \{(.*)\}$", d)
        if m:
            nxt = 0
            for item in m.group(1).split(","):
                item = item.strip()
                if not item:
                    continue
                if "=" in item:
                    name, v = [x.strip() for x in item.split("=")]
                    nxt = int(v, 0)
                else:
                    name = item
                consts.append((name, "i32", str(nxt)))
                nxt += 1
            continue
        m = re.match(r"^typedef struct (\w+) (\w+)$", d)
        if m:
            known.add(m.group(2))
            types.append("#[repr(C)]\npub struct %s {\n    _private: [u8; 0],\n}" % m.group(2))
            continue
        m = re.match(r"^typedef (\w+) (\w+)$", d)
        if m:
            known.add(m.group(2))
            types.append("pub type %s = %s;" % (m.group(2), SCALARS[m.group(1)]))
            continue
        m = re.match(r"^typedef struct (\w+) \{(.*)\} (\w+)$", d)
        if m:
            name = m.group(3)
            known.add(name)
            fields = []
            for f in m.group(2).split(";"):
                f = f.strip()
                if not f:
                    continue
                am = re.match(r"^(.*?)(\w+)\[(\d+)\]$", f)
                if am:
                    fields.append((ident(am.group(2)), "[%s; %s]" % (rust_type(am.group(1), known), am.group(3))))
                    continue
                if "," in f:   # `uint64_t a, b, c` (no pointers in such declarations in this header)
                    first, rest = f.split(",", 1)
                    fm = re.match(r"^(.*?)(\w+)$", first.strip())
                    assert "*" not in f
                    for nm in [fm.group(2)] + [x.strip() for x in rest.split(",")]:
                        fields.append((ident(nm), rust_type(fm.group(1), known)))
                    continue
                fm = re.match(r"^(.*?)(\w+)$", f)
                fields.append((ident(fm.group(2)), rust_type(fm.group(1), known)))
            structs.append((name, fields))
            continue
        m = re.match(r"^typedef (\w[\w \*]*?)\(\*(\w+)\)\((.*)\)$", d)
        if m:
            known.add(m.group(2))
            fnptrs.append((m.group(2), m.group(1).strip(), m.group(3)))
            continue
        m = re.match(r"^([\w \*]+?)\b(pcdn_\w+)\((.*)\)$", d)
        if m:
            funcs.append((m.group(2), m.group(1).strip(), m.group(3)))
            continue
        raise SystemExit("gen_pcdn_sys: cannot parse declaration: %r" % d)

    o = []
    o.append("//! pcdn-sys — raw FFI binding of `include/pcdn_fanout.h`, the C ABI of the H100 fan-out engine")
    o.append("//! (libpcdn_fanout.so).  GENERATED by scripts/gen_pcdn_sys.py from the header: do not edit;")
    o.append("//! tests/test_pcdn_sys.py fails when this file and the header diverge.  The meaning of every item,")
    o.append("//! and the reference function each entry point replaces, is documented in the header.")
    o.append("#![allow(non_camel_case_types, non_upper_case_globals, dead_code)]")
    o.append("")
    o.append("use std::os::raw::{c_char, c_int, c_void};")
    o.append("")
    for name, ty, v in consts:
        o.append("pub const %s: %s = %s;" % (name, ty, v))
    o.append("")
    for t in types:
        o.append(t)
        o.append("")
    for name, ret, params in fnptrs:
        ps = parse_params(params, known)
        r = "" if ret == "void" else " -> " + rust_type(ret, known)
        o.append("pub type %s = Option<unsafe extern \"C\" fn(%s)%s>;" % (name, ", ".join("%s: %s" % p for p in ps), r))
        o.append("")
    for name, fields in structs:
        o.append("#[repr(C)]\n#[derive(Clone, Copy)]\npub struct %s {" % name)
        for fn_, ft in fields:
            o.append("    pub %s: %s," % (fn_, ft))
        o.append("}")
        o.append("")
    o.append('#[link(name = "pcdn_fanout")]')
    o.append('extern "C" {')
    for name, ret, params in funcs:
        ps = parse_params(params, known)
        r = "" if ret == "void" else " -> " + rust_type(ret, known)
        o.append("    pub fn %s(%s)%s;" % (name, ", ".join("%s: %s" % p for p in ps), r))
    o.append("}")
    o.append("")
    return "\n".join(o), funcs


def main():
    text, _ = generate()
    if "--check" in sys.argv:
        cur = open(OUT).read() if os.path.exists(OUT) else ""
        if cur != text:
            sys.stderr.write("pcdn-sys/src/lib.rs is out of date: run python scripts/gen_pcdn_sys.py\n")
            sys.exit(1)
        return
    os.makedirs(os.path.dirname(OUT), exist_ok=True)
    with open(OUT, "w") as f:
        f.write(text)
    print("wrote", OUT)


if __name__ == "__main__":
    main()
