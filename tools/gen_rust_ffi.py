#!/usr/bin/env python
"""Generates bindings/rust/src/ffi.rs from include/qb200.h: every QB_API function as an `extern "C"` declaration, the POD structs,
the status / enum constants.  The Rust toolchain is absent from the build image, so the output is source only; regenerating it from
the header keeps it complete (tests/test_capi_symbols.py checks that it declares every exported function with the right arity)."""
import os
import re

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HDR = os.path.join(ROOT, "include", "qb200.h")
OUT = os.path.join(ROOT, "bindings", "rust", "src", "ffi.rs")

SCALARS = {"int32_t": "i32", "uint32_t": "u32", "uint64_t": "u64", "int64_t": "i64", "uint8_t": "u8", "size_t": "usize", "float": "f32", "double": "f64",
           "int": "i32", "qb_status": "qb_status", "char": "c_char", "void": "c_void"}
ENUMS = ("qb_distance", "qb_dtype", "qb_qdistance", "qb_bq_encoding", "qb_bq_query_encoding", "qb_query_kind", "qb_hnsw_algorithm", "qb_sparse_kind")
OPAQUE = ("qb_storage", "qb_scorer", "qb_hnsw", "qb_comm", "qb_sparse_index", "qb_sparse_storage")
STRUCTS = ("qb_scored_point", "qb_hw_counters")


def rust_type(c: str) -> str:
    c = re.sub(r"/\*.*?\*/", "", c).strip()
    c = c.replace("volatile", "").strip()
    stars = c.count("*")
    base = c.replace("*", " ")
    toks = base.split()
    const_first = toks and toks[0] == "const"
    words = [t for t in toks if t != "const"]
    name = words[0]
    inner_const = "const" in toks[1:] and stars == 2      # `T* const*`
    if name in ENUMS:
        r = "i32"
    elif name in OPAQUE or name in STRUCTS:
        r = name
    else:
        r = SCALARS[name]
    if stars == 0:
        return r
    if stars == 1:
        return f"*{'const' if const_first else 'mut'} {r}"
    if inner_const:
        return f"*const *mut {r}"
    return f"*mut *{'const' if const_first else 'mut'} {r}"


def parse():
    src = open(HDR).read()
    src_nc = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    fns = []
    for m in re.finditer(r"QB_API\s+([^;(]*?)\b(qb_[a-z0-9_]+)\s*\(([^;]*?)\)\s*;", src_nc, flags=re.S):
        ret, name, args = m.group(1).strip(), m.group(2), m.group(3).strip()
        params = []
        if args and args != "void":
            for a in [x.strip() for x in args.split(",")]:
                mm = re.match(r"(.*?)([A-Za-z_][A-Za-z0-9_]*)$", a, flags=re.S)
                params.append((mm.group(2), rust_type(mm.group(1))))
        fns.append((name, params, rust_type(ret) if ret != "void" else None))
    status = re.findall(r"(QB_(?:OK|ERR_[A-Z_]+))\s*=\s*(-?\d+)", src_nc)
    abi = re.search(r"#define QB200_ABI_VERSION (\d+)", src).group(1)
    return fns, status, abi


def main():
    fns, status, abi = parse()
    o = ["//! Raw FFI declarations for libqdrant_b200.so — GENERATED from include/qb200.h by tools/gen_rust_ffi.py; do not edit by hand.",
         "//! SOURCE ONLY: there is no Rust toolchain in the build image, so this file has never been compiled there; it is the binding a",
         "//! Qdrant maintainer would add under `lib/segment/src/vector_storage/b200/ffi.rs`.  One declaration per exported function.",
         "#![allow(non_camel_case_types)]", "use std::os::raw::{c_char, c_void};", "",
         "pub type qb_status = i32;", f"pub const QB200_ABI_VERSION: i32 = {abi};"]
    o += [f"pub const {k}: qb_status = {v};" for k, v in status]
    o += ["", "// Distance (types.rs:313-322), VectorStorageDatatype, quantization::DistanceType, BQ encodings, QueryVector kinds — passed as i32",
          "pub const QB_DIST_COSINE: i32 = 0; pub const QB_DIST_EUCLID: i32 = 1; pub const QB_DIST_DOT: i32 = 2; pub const QB_DIST_MANHATTAN: i32 = 3;",
          "pub const QB_DT_F32: i32 = 0; pub const QB_DT_F16: i32 = 1; pub const QB_DT_U8: i32 = 2;",
          "pub const QB_QD_COSINE: i32 = 0; pub const QB_QD_DOT: i32 = 1; pub const QB_QD_L1: i32 = 2; pub const QB_QD_L2: i32 = 3;",
          "// qb_hnsw_algorithm (SearchAlgorithm, graph_layers.rs:80-84)",
          "pub const QB_HNSW_ALGO_HNSW: i32 = 0; pub const QB_HNSW_ALGO_ACORN: i32 = 1;",
          "// qb_sparse_kind: InvertedIndexRam (may prune), the compressed indexes with f32 / f16 / u8 weights",
          "pub const QB_SPARSE_RAM: i32 = 0; pub const QB_SPARSE_COMPRESSED: i32 = 1; pub const QB_SPARSE_COMPRESSED_F16: i32 = 2; pub const QB_SPARSE_COMPRESSED_U8: i32 = 3;", ""]
    for name in OPAQUE:
        o += ["#[repr(C)]", f"pub struct {name} {{ _private: [u8; 0] }}"]
    o += ["", "/// Same layout as `common::types::ScoredPointOffset` (`#[repr(C)] { idx: u32, score: f32 }`).", "#[repr(C)]", "#[derive(Copy, Clone, Default, Debug, PartialEq)]",
          "pub struct qb_scored_point { pub idx: u32, pub score: f32 }", "", "#[repr(C)]", "#[derive(Copy, Clone, Default, Debug)]",
          "pub struct qb_hw_counters { pub cpu: u64, pub vector_io_read: u64 }", "", '#[link(name = "qdrant_b200")]', 'extern "C" {']
    for name, params, ret in fns:
        args = ", ".join(f"{('r#' + n) if n in ('type', 'ref', 'in') else n}: {t}" for n, t in params)
        o.append(f"    pub fn {name}({args}){' -> ' + ret if ret else ''};")
    o += ["}", ""]
    os.makedirs(os.path.dirname(OUT), exist_ok=True)
    open(OUT, "w").write("\n".join(o))
    return len(fns)


if __name__ == "__main__":
    print(main(), "functions ->", OUT)
