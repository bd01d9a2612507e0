"""A small baseline JPEG writer for test streams that neither zignal's encoder nor Pillow writes: 4:1:1, scans of one component, a
gray component with id != 1 and 2 x 2 sampling, restart intervals (with FF bytes before an RST, which end the scan), tables whose
codes all have one length, and symbol-level streams for the decoding details and error classes (semantic_cases).  Coefficients come in decode order (MCU by MCU, each MCU's blocks in scan order), in natural (row-major) order.
Plain Python: the streams are small."""
from __future__ import annotations

import numpy as np

ZIGZAG = [0, 1, 8, 16, 9, 2, 3, 10, 17, 24, 32, 25, 18, 11, 4, 5, 12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13, 6, 7, 14, 21, 28, 35, 42,
          49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63]
# T.81 Annex K tables K.3 (DC luma) and K.5 (AC luma)
DC_BITS = [0, 1, 5, 1, 1, 1, 1, 1, 1, 0, 0, 0, 0, 0, 0, 0]
DC_VALS = list(range(12))
AC_BITS = [0, 2, 1, 3, 3, 2, 4, 3, 5, 5, 4, 4, 0, 0, 1, 125]
AC_VALS = [
    0x01, 0x02, 0x03, 0x00, 0x04, 0x11, 0x05, 0x12, 0x21, 0x31, 0x41, 0x06, 0x13, 0x51, 0x61, 0x07, 0x22, 0x71, 0x14, 0x32, 0x81, 0x91,
    0xa1, 0x08, 0x23, 0x42, 0xb1, 0xc1, 0x15, 0x52, 0xd1, 0xf0, 0x24, 0x33, 0x62, 0x72, 0x82, 0x09, 0x0a, 0x16, 0x17, 0x18, 0x19, 0x1a,
    0x25, 0x26, 0x27, 0x28, 0x29, 0x2a, 0x34, 0x35, 0x36, 0x37, 0x38, 0x39, 0x3a, 0x43, 0x44, 0x45, 0x46, 0x47, 0x48, 0x49, 0x4a, 0x53,
    0x54, 0x55, 0x56, 0x57, 0x58, 0x59, 0x5a, 0x63, 0x64, 0x65, 0x66, 0x67, 0x68, 0x69, 0x6a, 0x73, 0x74, 0x75, 0x76, 0x77, 0x78, 0x79,
    0x7a, 0x83, 0x84, 0x85, 0x86, 0x87, 0x88, 0x89, 0x8a, 0x92, 0x93, 0x94, 0x95, 0x96, 0x97, 0x98, 0x99, 0x9a, 0xa2, 0xa3, 0xa4, 0xa5,
    0xa6, 0xa7, 0xa8, 0xa9, 0xaa, 0xb2, 0xb3, 0xb4, 0xb5, 0xb6, 0xb7, 0xb8, 0xb9, 0xba, 0xc2, 0xc3, 0xc4, 0xc5, 0xc6, 0xc7, 0xc8, 0xc9,
    0xca, 0xd2, 0xd3, 0xd4, 0xd5, 0xd6, 0xd7, 0xd8, 0xd9, 0xda, 0xe1, 0xe2, 0xe3, 0xe4, 0xe5, 0xe6, 0xe7, 0xe8, 0xe9, 0xea, 0xf1, 0xf2,
    0xf3, 0xf4, 0xf5, 0xf6, 0xf7, 0xf8, 0xf9, 0xfa]
# Every code one length: 12 DC codes of 4 bits, 162 AC codes of 8 bits (the decoder's worst case: a wrong bit phase never heals)
FLAT_DC_BITS = [0, 0, 0, 12] + [0] * 12
FLAT_AC_BITS = [0] * 7 + [162] + [0] * 8


def canonical(bits, vals):
    codes, code, k = {}, 0, 0
    for length in range(1, 17):
        for _ in range(bits[length - 1]):
            codes[vals[k]] = (code, length)
            code += 1
            k += 1
        code <<= 1
    return codes


class BitWriter:
    def __init__(self):
        self.out = bytearray()
        self.acc = 0
        self.n = 0

    def put(self, v, n):
        for i in range(n - 1, -1, -1):
            self.acc = (self.acc << 1) | ((v >> i) & 1)
            self.n += 1
            if self.n == 8:
                self.out.append(self.acc)
                if self.acc == 0xFF:
                    self.out.append(0)
                self.acc = self.n = 0

    def flush(self):
        while self.n:
            self.put(1, 1)


def _cat(v):
    return 0 if v == 0 else int(abs(int(v))).bit_length()


def _mag(v, c):
    return v if v >= 0 else v + (1 << c) - 1


def _segment(o, marker, payload):
    o += bytes([0xFF, marker]) + (len(payload) + 2).to_bytes(2, "big") + bytes(payload)


def write(width, height, comps, scan, mcus, qtables, dc_tables=None, ac_tables=None, restart=0, fill_ff_before_rst=0,
          raw_tail=b"", eoi=True):
    """comps: [(id, h, v, tq)]; scan: [(component id, td, ta)]; mcus: per MCU, a list of (scan component index, 64 natural coefs);
    qtables: {id: 64 natural values (< 256)}; tables: {id: (bits, vals)} (default: K.3 / K.5 as table 0)."""
    dc_tables = dc_tables or {0: (DC_BITS, DC_VALS)}
    ac_tables = ac_tables or {0: (AC_BITS, AC_VALS)}
    o = bytearray(b"\xFF\xD8")
    p = bytearray()
    for tid, q in qtables.items():
        p.append(tid)
        p += bytes(int(q[ZIGZAG[i]]) for i in range(64))
    _segment(o, 0xDB, p)
    p = bytearray([8]) + height.to_bytes(2, "big") + width.to_bytes(2, "big") + bytes([len(comps)])
    for cid, h, v, tq in comps:
        p += bytes([cid, h << 4 | v, tq])
    _segment(o, 0xC0, p)
    p = bytearray()
    for cls, tabs in ((0, dc_tables), (1, ac_tables)):
        for tid, (bits, vals) in tabs.items():
            p += bytes([cls << 4 | tid]) + bytes(bits) + bytes(vals)
    _segment(o, 0xC4, p)
    if restart:
        _segment(o, 0xDD, restart.to_bytes(2, "big"))
    p = bytearray([len(scan)])
    for cid, td, ta in scan:
        p += bytes([cid, td << 4 | ta])
    p += bytes([0, 63, 0])
    _segment(o, 0xDA, p)
    if mcus is None:   # header only (write_symbols)
        return o
    dcc = {k: canonical(*t) for k, t in dc_tables.items()}
    acc = {k: canonical(*t) for k, t in ac_tables.items()}
    w = BitWriter()
    pred = [0] * len(scan)
    for m, blocks in enumerate(mcus):
        if restart and m and m % restart == 0:
            w.flush()
            w.out += b"\xFF" * fill_ff_before_rst + bytes([0xFF, 0xD0 + (m // restart - 1) % 8])
            pred = [0] * len(scan)
        for si, coef in blocks:
            _, td, ta = scan[si]
            coef = [int(c) for c in np.asarray(coef).reshape(64)]
            diff = coef[0] - pred[si]
            pred[si] = coef[0]
            c = _cat(diff)
            code, ln = dcc[td][c]
            w.put(code, ln)
            w.put(_mag(diff, c), c)
            run = 0
            for k in range(1, 64):
                v = coef[ZIGZAG[k]]
                if v == 0:
                    run += 1
                    continue
                while run >= 16:
                    w.put(*acc[ta][0xF0])
                    run -= 16
                c = _cat(v)
                w.put(*acc[ta][run << 4 | c])
                w.put(_mag(v, c), c)
                run = 0
            if run:
                w.put(*acc[ta][0x00])
    w.flush()
    o += w.out + raw_tail
    if eoi:
        o += b"\xFF\xD9"
    return bytes(o)


def random_mcus(rng, n_mcus, blocks_per_mcu, scale=8, density=0.25):
    """MCUs of random coefficients: [(scan component index, coefs)], DC in [-60, 60], sparse small ACs."""
    out = []
    for _ in range(n_mcus):
        blocks = []
        for si in blocks_per_mcu:
            c = np.zeros(64, np.int32)
            c[0] = rng.integers(-60, 61)
            mask = rng.random(63) < density
            c[1:][mask] = rng.integers(-scale, scale + 1, mask.sum())
            blocks.append((si, c))
        out.append(blocks)
    return out


def write_symbols(width, height, comps, scan, mcus, qtables, dc_tables, ac_tables, eoi=True):
    """A stream whose entropy-coded segment is given symbol by symbol, so that it can hold what an encoder never writes (a run that
    reaches k = 64 with a size, DC categories above 11, AC symbols of size 0 with a run other than 0 or 15).  mcus: per MCU a list of
    (class 0 DC / 1 AC / None for raw bits alone, table id, symbol, raw bits value, raw bit count)."""
    o = write(width, height, comps, scan, None, qtables, dc_tables, ac_tables)
    codes = {(0, k): canonical(*t) for k, t in dc_tables.items()}
    codes.update({(1, k): canonical(*t) for k, t in ac_tables.items()})
    w = BitWriter()
    for syms in mcus:
        for cls, tid, sym, value, nbits in syms:
            if cls is not None:   # None: raw bits only
                w.put(*codes[(cls, tid)][sym])
            w.put(value, nbits)
    w.flush()
    o += w.out
    if eoi:
        o += b"\xFF\xD9"
    return bytes(o)


def block_symbols(coef, pred, tid=0):
    """The symbols of one ordinary block (DC difference to pred, then run / size pairs, ZRL, EOB) for write_symbols."""
    coef = [int(c) for c in np.asarray(coef).reshape(64)]
    diff = coef[0] - pred
    c = _cat(diff)
    out = [(0, tid, c, _mag(diff, c), c)]
    run = 0
    for k in range(1, 64):
        v = coef[ZIGZAG[k]]
        if v == 0:
            run += 1
            continue
        while run >= 16:
            out.append((1, tid, 0xF0, 0, 0))
            run -= 16
        c = _cat(v)
        out.append((1, tid, run << 4 | c, _mag(v, c), c))
        run = 0
    if run:
        out.append((1, tid, 0x00, 0, 0))
    return out


# Tables of the semantic cases: K.3 with DC category 11 replaced by 12 (InvalidDCCoefficient), K.5 with 0xFA replaced by 0x30 (size 0
# with run 3: InvalidACCoefficient).  Both stay complete prefix codes, so every other symbol decodes as usual.
SEM_DC = (DC_BITS, list(range(11)) + [12])
SEM_AC = (AC_BITS, AC_VALS[:-1] + [0x30])


def semantic_cases():
    """name -> (stream, expected status, expected reference error name or None).  One gray component with id 1, 64 x 32 pixels:
    32 blocks walked one by one.  Each case holds one of the details a textbook decoder gets wrong, or one error class, with a
    truncated twin where the data ends before the error (truncation comes first in decode order, so the call succeeds)."""
    rng = np.random.default_rng(64)
    n = 32
    coefs = []
    for _ in range(n):
        c = np.zeros(64, np.int32)
        c[0] = rng.integers(-60, 61)
        mask = rng.random(63) < 0.3
        c[1:][mask] = rng.integers(-20, 21, mask.sum())
        coefs.append(c)
    q = {0: np.full(64, 4)}
    comps, scan = [(1, 1, 1, 0)], [(1, 0, 0)]

    def blocks(special):
        out, pred = [], 0
        for b in range(n):
            if b in special:
                syms = special[b](pred)
            else:
                syms = block_symbols(coefs[b], pred)
                pred = int(coefs[b][0])
            out.append(syms)
        return out

    zrl3 = [(1, 0, 0xF0, 0, 0)] * 3   # k: 1 -> 49

    def run_to_64(pred):   # DC unchanged, k 49 + run 15 reaches 64: the block ends before the 5 magnitude bits
        return [(0, 0, 0, 0, 0)] + zrl3 + [(1, 0, 0xF5, 0, 0)]

    def zrl_clip(pred):    # a value at k = 49, then ZRL from k = 50 clipped at 64 (no EOB)
        return [(0, 0, 0, 0, 0)] + zrl3 + [(1, 0, 0x02, 3, 2), (1, 0, 0xF0, 0, 0)]

    def bad_dc(pred):
        return [(0, 0, 12, 0, 0)]

    def bad_ac(pred):
        return [(0, 0, 0, 0, 0), (1, 0, 0x30, 0, 0)]

    def bad_code(pred):    # sixteen 1-bits: no code of K.5 (its all-ones code is reserved)
        return [(0, 0, 0, 0, 0), (None, 0, 0, 0xFFFF, 16)]

    tabs = ({0: SEM_DC}, {0: SEM_AC})
    w = lambda mc, sc=scan, dc=tabs[0], ac=tabs[1], eoi=True: write_symbols(64, 32, comps, sc, mc, q, dc, ac, eoi=eoi)
    cases = {}
    cases["run_to_64"] = (w(blocks({3: run_to_64, 10: run_to_64, 21: run_to_64})), 0, None)
    cases["zrl_clip"] = (w(blocks({4: zrl_clip, 17: zrl_clip})), 0, None)
    for name, fn, at, err in (("invalid_dc", bad_dc, 12, "InvalidDCCoefficient"), ("invalid_ac", bad_ac, 7, "InvalidACCoefficient"),
                              ("invalid_code", bad_code, 20, "InvalidHuffmanCode")):
        full = blocks({at: fn})
        cases[name] = (w(full), 31, err)
        cases[name + "_after_truncation"] = (w(full[:at], eoi=False), 0, None)
    ordinary = blocks({})
    cases["ordinary"] = (w(ordinary), 0, None)
    cases["missing_ac_table"] = (w(ordinary, sc=[(1, 0, 1)]), 31, "MissingHuffmanTable")
    cases["missing_ac_table_after_truncation"] = (w([], sc=[(1, 0, 1)]), 0, None)   # the DC read runs out first
    cases["missing_dc_table_no_data"] = (w([], sc=[(1, 1, 0)]), 31, "MissingHuffmanTable")   # checked before any read
    # only the first scan is decoded: a second SOS with other data changes nothing
    first = w(ordinary, eoi=False)
    second = write_symbols(64, 32, comps, scan, blocks({}), q, *tabs, eoi=True)
    cases["two_scans"] = (first + second[second.index(b"\xFF\xDA"):], 0, None)
    return cases
