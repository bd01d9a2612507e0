#!/usr/bin/env python
"""Regenerates the `extern fn` block of zig/zignal_b200.zig from include/zignal_b200.h, so the Zig side of the boundary declares
every entry point of the C ABI with matching types.  `--check` exits 1 if the block is stale (tests/test_zig_shim.py runs it).

usage: python tools/gen_zig_externs.py [--check]
"""
import re
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
HEADER = ROOT / "include" / "zignal_b200.h"
ZIG = ROOT / "zig" / "zignal_b200.zig"
BEGIN = "    // ---- BEGIN GENERATED (tools/gen_zig_externs.py from include/zignal_b200.h) ----"
END = "    // ---- END GENERATED ----"

OPAQUE = {"zb_fdm": "Fdm", "zb_shard_comm": "ShardComm", "zb_shard_image": "ShardImage", "zb_hough": "Hough"}
STRUCTS = {"zb_hough_line": "HoughLine", "zb_diff_stats": "DiffStats", "zb_jpeg_options": "JpegOptions", "zb_jpeg_limits": "JpegLimits",
           "zb_jpeg_header": "JpegHeader", "zb_color_image": "ColorImage"}   # extern structs other than zb_image
SCALARS = {"int": "c_int", "int32_t": "i32", "uint32_t": "u32", "uint64_t": "u64", "size_t": "usize", "float": "f32", "double": "f64",
           "uint8_t": "u8", "uint16_t": "u16", "zb_stream": "Stream"}
# pointer parameters that are single out-values rather than arrays: (function, parameter) or parameter name alone
SINGLE_OUT = {"count", "ordinal", "n", "out_rows", "out_cols", "converged", "rank", "world", "peer_access", "lo", "hi", "interior_first", "threshold",
              "bytes", "len", "sign", "det", ("zb_diff", "stats"), ("zb_jpeg_info", "out")}
# per-file arrays of a batch call, where the name alone would read as a single value or a single image
BATCH = {("zb_jpeg_decode_batch", "data"): "[*]const [*]const u8", ("zb_jpeg_decode_batch", "len"): "[*]const u64",
         ("zb_jpeg_decode_batch", "dst"): "[*]ZbImage"}


def zig_type(ctype: str, name: str, fn: str) -> str:
    t = " ".join(ctype.split())
    const = t.startswith("const ")
    base = t[6:] if const else t
    stars = base.count("*")
    base = base.replace("*", "").strip()
    if stars == 0:
        return SCALARS[base]
    if base == "zb_image":
        return "*const ZbImage" if const else "*ZbImage"
    if base in OPAQUE:
        return f"*?*{OPAQUE[base]}" if stars == 2 else f"?*{OPAQUE[base]}"
    if base == "void":
        return "*?*anyopaque" if stars == 2 else "*const anyopaque" if const else "?*anyopaque"
    if base == "char":
        return "[*:0]const u8"
    if base == "zb_stream":
        return "*Stream"
    if base in STRUCTS:
        if base == "zb_jpeg_limits":
            return "?*const JpegLimits"           # NULL: the reference's DecodeLimits defaults
        if const:
            return f"*const {STRUCTS[base]}"   # one input (zb_jpeg_encode's options, zb_convert_color's source)
        if base == "zb_color_image":
            return "*ColorImage"                  # zb_convert_color's destination
        if (fn, name) in SINGLE_OUT:
            return f"?*{STRUCTS[base]}"  # one optional result (zb_diff's stats, NULL for none)
        return f"?[*]{STRUCTS[base]}"   # may be NULL when the capacity is 0 (zb_hough_find_lines)
    if fn == "zb_hough_create" and name in ("cos_table", "sin_table"):
        return "?[*]const i32"          # NULL: the library computes the tables
    z = SCALARS[base]
    if name in SINGLE_OUT or (name == "out" and fn in ("zb_psnr", "zb_ssim", "zb_mean_pixel_error")):
        return f"*{z}"
    if fn.startswith("zb_gemm") and name == "c":
        return f"?[*]const {z}"   # Matrix.gemm's optional C (Matrix.zig:709)
    if fn.startswith("zb_svd_dev") and name in ("d_u", "d_v"):
        return f"?[*]{z}"
    if fn.startswith("zb_center_columns") and name == "centered":
        return f"?[*]{z}"
    if fn == "zb_shard_comm_create" and name == "id128":
        return "?[*]const u8"
    return f"[*]const {z}" if const else f"?[*]{z}" if fn.startswith("zb_svd") or fn.startswith("zb_shard_comm_info") else f"[*]{z}"


def prototypes():
    text = HEADER.read_text()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    text = re.sub(r"^\s*#.*$", "", text, flags=re.M)
    out = []
    for m in re.finditer(r"\b(int|uint64_t|const char\*)\s+(zb_[a-z0-9_]+)\s*\(([^;{}]*?)\)\s*;", text, flags=re.S):
        ret, fn, args = m.group(1), m.group(2), " ".join(m.group(3).split())
        params = []
        if args and args != "void":
            for a in args.split(","):
                a = a.strip()
                mm = re.match(r"(.*?)([A-Za-z_][A-Za-z0-9_]*)$", a)
                ctype, name = mm.group(1).strip(), mm.group(2)
                params.append((ctype, name))
        out.append((ret, fn, params))
    return out


def render():
    lines = [BEGIN]
    for ret, fn, params in prototypes():
        zret = {"int": "c_int", "uint64_t": "u64", "const char*": "[*:0]const u8"}[ret]
        zparams = []
        for ctype, name in params:
            zname = {"self": "self_", "error": "err", "type": "type_", "c": "c_"}.get(name, name)   # `c` would shadow the container
            zt = BATCH.get((fn, name)) or zig_type(ctype, name, fn)
            if fn == "zb_shard_comm_info" and name in ("rank", "world", "peer_access"):
                zt = "?*c_int"
            if fn.startswith("zb_svd") and name == "converged":
                zt = "?*u64"
            if fn.startswith("zb_svd") and name == "a":
                zt = zt.replace("?[*]", "[*]")
            zparams.append(f"{zname}: {zt}")
        lines.append(f"    pub extern fn {fn}({', '.join(zparams)}) {zret};")
    lines.append(END)
    return "\n".join(lines)


def main():
    src = ZIG.read_text()
    a, b = src.index(BEGIN), src.index(END) + len(END)
    new = src[:a] + render() + src[b:]
    if "--check" in sys.argv:
        if new != src:
            print("zig/zignal_b200.zig: extern block is stale; run tools/gen_zig_externs.py")
            sys.exit(1)
        return
    ZIG.write_text(new)
    print(f"{len(prototypes())} entry points declared")


if __name__ == "__main__":
    main()
