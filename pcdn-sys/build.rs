// build.rs — tells cargo where libpcdn_fanout.so lives.
//
// PCDN_LIB_DIR: directory that holds libpcdn_fanout.so (default: ../push-cdn_b200 relative to this
// crate, where `python -c 'import __graft_entry__ as g; g.build()'` leaves it).  The library is built
// by nvcc for sm_90a; this script does not compile anything.
use std::{env, path::PathBuf};

fn main() {
    let dir = env::var("PCDN_LIB_DIR").map(PathBuf::from).unwrap_or_else(|_| {
        PathBuf::from(env::var("CARGO_MANIFEST_DIR").unwrap()).join("..").join("push-cdn_b200")
    });
    println!("cargo:rustc-link-search=native={}", dir.display());
    println!("cargo:rustc-link-lib=dylib=pcdn_fanout");
    println!("cargo:rustc-link-arg=-Wl,-rpath,{}", dir.display());
    println!("cargo:rerun-if-env-changed=PCDN_LIB_DIR");
    println!("cargo:rerun-if-changed=build.rs");
}
