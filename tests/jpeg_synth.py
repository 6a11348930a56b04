"""Synthetic JPEG files for the tests of the device decoder (csrc/jpeg_decode.cu), and a plain-integer restatement of
the decode cv2.imread does on them.

No encoder writes the streams these tests need: coefficients past 11 bits, quantisers up to 65535, DC predictors that
leave int16, 16-bit codes, scans whose subsequences never self-synchronise.  So:

- `write` codes given quantised coefficients with given tables (DQT 8- or 16-bit, any DHT, DRI / RSTn, 1 or 3
  components at 4:4:4 / 4:2:2 / 4:2:0, ZRL runs, byte stuffing) into a SOF0 or SOF1 file;
- `decode` restates what cv2.imread returns for such a file, in Python integers and numpy: the Huffman parse into int16
  coefficients with libjpeg's int DC predictor, the islow IDCT in the 16-bit lanes of libjpeg-turbo's x86 SIMD code
  (jsimd_idct_islow), jdsample.c's fancy upsampling and jdcolor.c's YCbCr -> BGR; it also reports, per block, which
  16-bit wraps and saturations the IDCT met;
- `sync_model` restates the device's synchronisation of subsequence entry states (the sync kernel and its host loop)
  and says how many launches and host rounds the iteration needs, and whether guessed states ever meet the true ones.

tests/test_jpeg_synth_cpu.py pins `write` and `decode` against OpenCV; tests/test_gpu_jpeg_decode_extreme.py holds the
device to both."""
import struct

import numpy as np

# zig-zag index -> natural (row-major) index
NATURAL = [0, 1, 8, 16, 9, 2, 3, 10, 17, 24, 32, 25, 18, 11, 4, 5, 12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13, 6, 7, 14,
           21, 28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53,
           60, 61, 54, 47, 55, 62, 63]
SAMPLING_HV = {"gray": (1, 1), "444": (1, 1), "422": (2, 1), "420": (2, 2)}
SUB_BITS, SYNC_HOPS, SYNC_LAUNCHES_PER_READ = 8192, 32, 4   # jpeg_decode.cu kSubBits, kSyncHops, kSyncLaunchesPerRead
ZRL, EOB = 0xF0, 0x00


def category(v):
    return int(abs(int(v))).bit_length()


def wrap16(v):
    return ((v + 32768) & 0xFFFF) - 32768


class Huff(object):
    """A Huffman table from [(symbol, code length)] in table order: canonical codes, shorter lengths first, and within a
    length the order given.  A symbol may be listed more than once (it is coded with its first code).  jdhuff.c's rules
    hold: at most 256 codes, and the all-ones code of every length stays unused."""

    def __init__(self, entries):
        assert 0 < len(entries) <= 256
        order = sorted(range(len(entries)), key=lambda i: (entries[i][1], i))
        self.bits = [0] * 16
        for _, length in entries:
            assert 1 <= length <= 16
            self.bits[length - 1] += 1
        self.vals = [entries[i][0] for i in order]
        self.enc = {}
        code, i = 0, 0
        for length in range(1, 17):
            for _ in range(self.bits[length - 1]):
                sym = self.vals[i]
                self.enc.setdefault(sym, (code, length))
                code += 1
                i += 1
            assert code < (1 << length), "the all-ones code of length %d would be used" % length
            code <<= 1

    @staticmethod
    def flat(symbols, length=8, long_symbols=(), long_length=16):
        """`symbols` with codes of `length` bits, then `long_symbols` with codes of `long_length` bits."""
        return Huff([(s, length) for s in symbols] + [(s, long_length) for s in long_symbols])

    def dht(self, tc, th):
        return bytes([(tc << 4) | th]) + bytes(self.bits) + bytes(self.vals)


def ac_symbols():
    """Every AC symbol: (run, category) for runs 0..15 and categories 1..15, ZRL and EOB (242 symbols)."""
    return [EOB, ZRL] + [(r << 4) | s for r in range(16) for s in range(1, 16)]


def standard_tables():
    """(dc, ac): every DC category and every AC symbol with 8-bit codes, the rest of the code space unused."""
    return Huff.flat(range(16)), Huff.flat(ac_symbols())


def _seg(marker, body):
    return bytes([0xFF, marker]) + struct.pack(">H", len(body) + 2) + body


class _BitWriter(object):
    def __init__(self):
        self.parts = []

    def put(self, code, n):
        if n:
            self.parts.append(format(code, "0%db" % n))

    def flush(self):
        """The bits so far padded with 1s to a byte, stuffed."""
        s = "".join(self.parts)
        self.parts = []
        s += "1" * (-len(s) % 8)
        if not s:
            return b""
        return int(s, 2).to_bytes(len(s) // 8, "big").replace(b"\xFF", b"\xFF\x00")


def mcu_shape(width, height, sampling):
    h, v = SAMPLING_HV[sampling]
    return (height + 8 * v - 1) // (8 * v), (width + 8 * h - 1) // (8 * h)


def plane_shapes(width, height, sampling):
    """[(block rows, block columns)] of each component's coefficient array (the MCU-padded planes)."""
    my, mx = mcu_shape(width, height, sampling)
    if sampling == "gray":
        return [(my, mx)]
    h, v = SAMPLING_HV[sampling]
    return [(my * v, mx * h), (my, mx), (my, mx)]


def write(planes, width, height, sampling, quant, dc, ac, restart=0, zrl_tail=False, sof=None):
    """A JPEG file holding `planes`: per component an int array (block rows, block columns, 64) in natural order, shaped
    as plane_shapes() says.  AC values lie in [-32767, 32767]; element 0 of a block is the DC predictor's value (any
    int: the stream codes the differences, which must lie in [-32767, 32767]; the decoder stores it modulo 2^16).
    quant[c] (64 values, natural order, 1..65535), dc[c] and ac[c] (Huff) are component c's tables.  restart: the restart
    interval in MCUs (0: none).  zrl_tail: a block whose trailing zeros are a multiple of 16 ends with ZRLs reaching
    k = 64 instead of an EOB.  sof: 0xC0 or 0xC1 (default: 0xC1 when a quantiser exceeds 255)."""
    ncomp = len(planes)
    assert ncomp == (1 if sampling == "gray" else 3)
    shapes = plane_shapes(width, height, sampling)
    for c in range(ncomp):
        assert planes[c].shape == shapes[c] + (64,), (c, planes[c].shape, shapes[c])
    hmax, vmax = SAMPLING_HV[sampling]
    my, mx = mcu_shape(width, height, sampling)
    wide = any(int(q) > 255 for qt in quant for q in qt)
    if sof is None:
        sof = 0xC1 if wide else 0xC0
    head = b"\xFF\xD8" + _seg(0xE0, b"JFIF\x00\x01\x01\x00\x00\x01\x00\x01\x00\x00")
    for c in range(ncomp):
        q = [int(quant[c][NATURAL[k]]) for k in range(64)]
        assert all(1 <= x <= 65535 for x in q)
        pq = 1 if max(q) > 255 else 0
        head += _seg(0xDB, bytes([(pq << 4) | c]) + b"".join(struct.pack(">H" if pq else ">B", x) for x in q))
    comps = b"".join(bytes([c + 1, ((hmax << 4) | vmax) if c == 0 else 0x11, c]) for c in range(ncomp))
    head += _seg(sof, bytes([8]) + struct.pack(">HH", height, width) + bytes([ncomp]) + comps)
    for c in range(ncomp):
        head += _seg(0xC4, dc[c].dht(0, c) + ac[c].dht(1, c))
    if restart:
        head += _seg(0xDD, struct.pack(">H", restart))
    head += _seg(0xDA, bytes([ncomp]) + b"".join(bytes([c + 1, (c << 4) | c]) for c in range(ncomp)) + b"\x00\x3F\x00")

    layout = [(0, dy, dx) for dy in range(vmax) for dx in range(hmax)] if ncomp == 3 else [(0, 0, 0)]
    layout += [(1, 0, 0), (2, 0, 0)] if ncomp == 3 else []
    bw, scan, pred = _BitWriter(), [], [0] * ncomp
    for m in range(my * mx):
        if restart and m and m % restart == 0:
            scan.append(bw.flush())
            scan.append(bytes([0xFF, 0xD0 + (m // restart - 1) % 8]))
            pred = [0] * ncomp
        y, x = divmod(m, mx)
        for c, dy, dx in layout:
            blk = planes[c][y * vmax + dy, x * hmax + dx] if c == 0 else planes[c][y, x]
            zz = [int(blk[NATURAL[k]]) for k in range(64)]
            d = zz[0] - pred[c]
            pred[c] = zz[0]
            s = category(d)
            assert s <= 15, "DC difference %d" % d
            bw.put(*dc[c].enc[s])
            bw.put(d if d >= 0 else d + (1 << s) - 1, s)
            nz = [k for k in range(1, 64) if zz[k]]
            last = nz[-1] if nz else 0
            run = 0
            for k in range(1, last + 1):
                if zz[k] == 0:
                    run += 1
                    continue
                while run > 15:
                    bw.put(*ac[c].enc[ZRL])
                    run -= 16
                s = category(zz[k])
                assert s <= 15, "AC value %d" % zz[k]
                bw.put(*ac[c].enc[(run << 4) | s])
                bw.put(zz[k] if zz[k] >= 0 else zz[k] + (1 << s) - 1, s)
                run = 0
            if last < 63:
                if zrl_tail and (63 - last) % 16 == 0:
                    for _ in range((63 - last) // 16):
                        bw.put(*ac[c].enc[ZRL])
                else:
                    bw.put(*ac[c].enc[EOB])
    scan.append(bw.flush())
    return head + b"".join(scan) + b"\xFF\xD9"


# ---- the restatement of the decode ------------------------------------------------------------------------------------
class _Table(object):
    """A decoding table: look[next 16 bits] = (code length, symbol), or None where no code starts."""

    def __init__(self, bits, vals):
        self.look = [None] * 65536
        code, p = 0, 0
        for length in range(1, 17):
            for _ in range(bits[length - 1]):
                lo = code << (16 - length)
                self.look[lo:lo + (1 << (16 - length))] = [(length, vals[p])] * (1 << (16 - length))
                code += 1
                p += 1
            code <<= 1


class Frame(object):
    """A file's header, and its scan unstuffed into one bit string (segment starts in bits)."""

    def __init__(self, f):
        assert f[:2] == b"\xFF\xD8"
        quant, dct, act, self.restart, i = {}, {}, {}, 0, 2
        while True:
            assert f[i] == 0xFF
            m = f[i + 1]
            n = struct.unpack(">H", f[i + 2:i + 4])[0]
            p = f[i + 4:i + 2 + n]
            if m in (0xC0, 0xC1):
                self.sof = m
                self.height, self.width = struct.unpack(">HH", p[1:5])
                self.ncomp = p[5]
                self.hv = [(p[7 + 3 * c] >> 4, p[7 + 3 * c] & 15) for c in range(self.ncomp)]
                self.tq = [p[8 + 3 * c] for c in range(self.ncomp)]
            elif m == 0xDB:
                o = 0
                while o < len(p):
                    pq, tq = p[o] >> 4, p[o] & 15
                    q = [0] * 64
                    for k in range(64):
                        q[NATURAL[k]] = struct.unpack(">H", p[o + 1 + 2 * k:o + 3 + 2 * k])[0] if pq else p[o + 1 + k]
                    quant[tq] = np.array(q, np.int64)
                    o += 1 + 64 * (pq + 1)
            elif m == 0xC4:
                o = 0
                while o < len(p):
                    bits = list(p[o + 1:o + 17])
                    n_sym = sum(bits)
                    (act if p[o] >> 4 else dct)[p[o] & 15] = _Table(bits, list(p[o + 17:o + 17 + n_sym]))
                    o += 17 + n_sym
            elif m == 0xDD:
                self.restart = struct.unpack(">H", p)[0]
            elif m == 0xDA:
                sel = [(p[2 + 2 * c] >> 4, p[2 + 2 * c] & 15) for c in range(p[0])]
                i += 2 + n
                break
            i += 2 + n
        self.hmax, self.vmax = (self.hv[0] if self.ncomp == 3 else (1, 1))
        self.quant = [quant[self.tq[c]] for c in range(self.ncomp)]
        self.dc = [dct[sel[c][0]] for c in range(self.ncomp)]
        self.ac = [act[sel[c][1]] for c in range(self.ncomp)]
        self.mcus_y = (self.height + 8 * self.vmax - 1) // (8 * self.vmax)
        self.mcus_x = (self.width + 8 * self.hmax - 1) // (8 * self.hmax)
        self.n_mcu = self.mcus_x * self.mcus_y
        self.blk_comp = [0] * (self.hmax * self.vmax) + ([1, 2] if self.ncomp == 3 else [])
        self.bpm = len(self.blk_comp)
        self.ri = self.restart or self.n_mcu
        # unstuff: 0xFF 0x00 -> 0xFF, RSTn starts the next segment, any other marker ends the scan
        out, starts, j = bytearray(), [0], i
        while j < len(f):
            b = f[j]
            if b != 0xFF:
                out.append(b)
                j += 1
                continue
            nxt = f[j + 1]
            if nxt == 0x00:
                out.append(0xFF)
                j += 2
            elif 0xD0 <= nxt <= 0xD7:
                starts.append(len(out))
                j += 2
            elif nxt == 0xFF:
                j += 1
            else:
                break
        n_seg = (self.n_mcu + self.ri - 1) // self.ri
        assert len(starts) >= n_seg
        self.seg_bytes = starts[:n_seg] + [starts[n_seg] if len(starts) > n_seg else len(out)]
        self.scan_bytes = len(out)
        # bytes past the end read as 0, as the device reads them
        self.bits = "".join(format(b, "08b") for b in out) + "0" * 64

    def step(self, pos, j, k):
        """decode_step: one codeword of block j at zig-zag index k from bit `pos`.  (pos, j, k, kout, value), kout 0 for
        a DC difference, the index of a non-zero AC coefficient, or -1; None for a code no table holds or a run past
        coefficient 63."""
        c = self.blk_comp[j]
        bits = self.bits
        kout, v = -1, 0
        if k == 0:
            e = self.dc[c].look[int(bits[pos:pos + 16], 2)]
            if e is None or e[1] > 15:
                return None
            pos += e[0]
            s = e[1]
            if s:
                r = int(bits[pos:pos + s], 2)
                v = r - (1 << s) + 1 if r < (1 << (s - 1)) else r
                pos += s
            kout, k = 0, 1
        else:
            e = self.ac[c].look[int(bits[pos:pos + 16], 2)]
            if e is None:
                return None
            pos += e[0]
            r, s = e[1] >> 4, e[1] & 15
            if s:
                k += r
                if k > 63:
                    return None
                x = int(bits[pos:pos + s], 2)
                v = x - (1 << s) + 1 if x < (1 << (s - 1)) else x
                pos += s
                kout = k
                k += 1
            elif r == 15:
                k += 16
                if k > 64:
                    return None
            else:
                k = 64
        if k == 64:
            k = 0
            j = j + 1 if j + 1 < self.bpm else 0
        return pos, j, k, kout, v

    def coefficients(self):
        """Per component the int16 coefficient array (block rows, block columns, 64) in natural order, the int DC
        predictor of each block (same shape without the 64), and the bit each block starts at."""
        shapes = [(self.mcus_y * self.vmax, self.mcus_x * self.hmax)] + [(self.mcus_y, self.mcus_x)] * (self.ncomp - 1)
        coef = [np.zeros(s + (64,), np.int64) for s in shapes]
        pred_of = [np.zeros(s, np.int64) for s in shapes]
        start_of = [np.zeros(s, np.int64) for s in shapes]
        layout = [(0, dy, dx) for dy in range(self.vmax) for dx in range(self.hmax)] + [(1, 0, 0), (2, 0, 0)]
        layout = layout[:self.bpm]
        for s in range(len(self.seg_bytes) - 1):
            pos, j, k = 8 * self.seg_bytes[s], 0, 0
            pred = [0] * self.ncomp
            for m in range(s * self.ri, min((s + 1) * self.ri, self.n_mcu)):
                y, x = divmod(m, self.mcus_x)
                for jb, (c, dy, dx) in enumerate(layout):
                    at = (y * self.vmax + dy, x * self.hmax + dx) if c == 0 else (y, x)
                    blk = coef[c][at]
                    start_of[c][at] = pos
                    while True:
                        r = self.step(pos, j, k)
                        assert r is not None, "corrupt scan"
                        pos, j, k, kout, v = r
                        if kout == 0:
                            pred[c] += v
                            pred_of[c][at] = pred[c]
                            blk[0] = wrap16(pred[c])
                        elif kout > 0:
                            blk[NATURAL[kout]] = v
                        if k == 0:
                            break
            assert pos <= 8 * self.seg_bytes[s + 1], "segment %d short of bits" % s
        return [c.astype(np.int16) for c in coef], pred_of, start_of


_M = 0xFFFFFFFF


def _w16(x):
    return ((x + 32768) & 0xFFFF) - 32768


def _out16(x):
    return (x < -32768) | (x > 32767)


def _i32(x):
    x = x & _M
    return np.where(x >= (1 << 31), x - (1 << 32), x)


def _idct_pass(v, sh, flags):
    """jpeg_decode.cu idct_pass on 8 int64 arrays of 16-bit values (32-bit lanes modulo 2^32, descale by sh)."""
    def mul(a, c):
        return (a * c) & _M
    z2, z3 = v[2], v[6]
    tmp3 = (mul(z2, 4433 + 6270) + mul(z3, 4433)) & _M
    tmp2 = (mul(z2, 4433) + mul(z3, 4433 - 15137)) & _M
    flags["even_wrap"] |= _out16(v[0] + v[4]) | _out16(v[0] - v[4])
    t0 = (_w16(v[0] + v[4]) << 13) & _M
    t1 = (_w16(v[0] - v[4]) << 13) & _M
    tmp10, tmp13, tmp11, tmp12 = (t0 + tmp3) & _M, (t0 - tmp3) & _M, (t1 + tmp2) & _M, (t1 - tmp2) & _M
    o0, o1, o2, o3 = v[7], v[5], v[3], v[1]
    flags["odd_wrap"] |= _out16(o0 + o2) | _out16(o1 + o3)
    z3o, z4o = _w16(o0 + o2), _w16(o1 + o3)
    za = (mul(z3o, 9633 - 16069) + mul(z4o, 9633)) & _M
    zb = (mul(z3o, 9633) + mul(z4o, 9633 - 3196)) & _M
    a0 = (mul(o0, 2446 - 7373) + mul(o3, -7373) + za) & _M
    a3 = (mul(o0, -7373) + mul(o3, 12299 - 7373) + zb) & _M
    a1 = (mul(o1, 16819 - 20995) + mul(o2, -20995) + zb) & _M
    a2 = (mul(o1, -20995) + mul(o2, 25172 - 20995) + za) & _M
    r = 1 << (sh - 1)
    out = [None] * 8
    for i, a, b, sg in ((0, tmp10, a3, 1), (7, tmp10, a3, -1), (1, tmp11, a2, 1), (6, tmp11, a2, -1),
                        (2, tmp12, a1, 1), (5, tmp12, a1, -1), (3, tmp13, a0, 1), (4, tmp13, a0, -1)):
        out[i] = _i32(a + sg * b + r) >> sh
    return out


IDCT_FLAGS = ("deq_wrap", "deq_max", "deq_min", "even_wrap", "odd_wrap", "pass1_sat", "shortcut", "shortcut_row0_ac",
              "shortcut_wrap", "clamp_lo", "clamp_hi")


def idct(coef, q):
    """(samples uint8 (n, 8, 8), {flag: bool (n,)}) of n blocks of int16 coefficients (n, 64) in natural order with the
    quantisers q (64, natural order), as jpeg_decode.cu's jdec_idct_kernel computes them.  The flags say which 16-bit
    wraps and saturations each block meets: deq_wrap a dequantised product outside int16, deq_max / deq_min one exactly
    at 32767 / -32768; even_wrap in0 +- in4 and odd_wrap z3 / z4 (in7 + in3, in5 + in1) wrapping in either pass;
    pass1_sat a pass-1 output saturated; shortcut the rows-1..7-are-zero path, shortcut_row0_ac with row-0 AC terms,
    shortcut_wrap with DC * q * 4 outside int16; clamp_lo / clamp_hi an output sample clamped at 0 / 255."""
    c = coef.astype(np.int64).reshape(-1, 64)
    n = c.shape[0]
    prod = c * np.asarray(q, np.int64)[None, :]
    f = {k: np.zeros(n, bool) for k in IDCT_FLAGS}
    f["deq_wrap"] = _out16(prod).any(1)
    f["deq_max"] = (prod == 32767).any(1)
    f["deq_min"] = (prod == -32768).any(1)
    deq = _w16(prod).reshape(n, 8, 8)
    short = ~(c[:, 8:] != 0).any(1)
    f["shortcut"] = short
    f["shortcut_row0_ac"] = short & (c[:, 1:8] != 0).any(1)
    f["shortcut_wrap"] = short & _out16(deq[:, 0, 0] * 4)
    pass_flags = {"even_wrap": np.zeros((n, 8), bool), "odd_wrap": np.zeros((n, 8), bool)}
    cols = _idct_pass([deq[:, r, :] for r in range(8)], 11, pass_flags)   # each (n, 8 columns)
    for k in ("even_wrap", "odd_wrap"):
        f[k] |= pass_flags[k].any(1) & ~short
    p1 = np.stack(cols, axis=1)                                         # (n, row, column)
    f["pass1_sat"] = _out16(p1).any((1, 2)) & ~short
    ws = np.where(short[:, None, None], _w16(deq[:, 0:1, :] * 4), np.clip(p1, -32768, 32767))
    pass_flags = {"even_wrap": np.zeros((n, 8), bool), "odd_wrap": np.zeros((n, 8), bool)}
    rows = _idct_pass([ws[:, :, x] for x in range(8)], 18, pass_flags)  # each (n, 8 rows)
    for k in ("even_wrap", "odd_wrap"):
        f[k] |= pass_flags[k].any(1)
    o = np.stack(rows, axis=2)                                          # (n, row, column)
    f["clamp_lo"] = (o < -128).any((1, 2))
    f["clamp_hi"] = (o > 127).any((1, 2))
    return (np.clip(o, -128, 127) + 128).astype(np.uint8), f


def _upsample(p, cw, ch, hr, vr, width, height):
    """jdsample.c's fancy upsampling of the chroma plane p (cw x ch samples) to width x height, as the device does it."""
    p = p.astype(np.int64)
    x = np.arange(width)[None, :]
    y = np.arange(height)[:, None]
    cx, cy = x // hr, y // vr
    if (hr == 1 and vr == 1) or cw <= 2:
        return p[cy, cx]
    def at(yy, xx):
        return p[yy, np.clip(xx, 0, cw - 1)]
    dx = np.where(x & 1, 1, -1)
    if vr == 1:
        return (at(cy, cx) * 3 + at(cy, cx + dx) + np.where(x & 1, 2, 1)) >> 2
    far = np.clip(cy + np.where(y & 1, 1, -1), 0, ch - 1)
    s0 = at(cy, cx) * 3 + at(far, cx)
    s1 = at(cy, cx + dx) * 3 + at(far, cx + dx)
    return (s0 * 3 + s1 + np.where(x & 1, 7, 8)) >> 4


def decode(f, channels):
    """(image, info) for the file f: the image cv2.imread returns (channels 1: gray, 3: B, G, R), and info: 'frame'
    (Frame), 'coef' / 'pred' / 'start' (Frame.coefficients), 'flags' ({flag: number of blocks}, over every component's
    blocks) and 'block_flags' (per component {flag: bool array shaped like its blocks})."""
    F = Frame(f)
    coef, pred, start = F.coefficients()
    planes, totals, per = [], {k: 0 for k in IDCT_FLAGS}, []
    for c in range(F.ncomp):
        by, bx = coef[c].shape[:2]
        s, fl = idct(coef[c].reshape(-1, 64), F.quant[c])
        planes.append(s.reshape(by, bx, 8, 8).transpose(0, 2, 1, 3).reshape(by * 8, bx * 8))
        per.append({k: v.reshape(by, bx) for k, v in fl.items()})
        for k in IDCT_FLAGS:
            totals[k] += int(fl[k].sum())
    info = dict(frame=F, coef=coef, pred=pred, start=start, flags=totals, block_flags=per)
    w, h = F.width, F.height
    Y = planes[0][:h, :w].astype(np.int64)
    if channels == 1:
        return Y.astype(np.uint8), info
    if F.ncomp == 1:
        return np.repeat(Y[:, :, None], 3, axis=2).astype(np.uint8), info
    cw, ch = (w + F.hmax - 1) // F.hmax, (h + F.vmax - 1) // F.vmax
    cb = _upsample(planes[1], cw, ch, F.hmax, F.vmax, w, h) - 128
    cr = _upsample(planes[2], cw, ch, F.hmax, F.vmax, w, h) - 128
    r = Y + ((91881 * cr + 32768) >> 16)
    g = Y + ((-22554 * cb + 32768 - 46802 * cr) >> 16)
    b = Y + ((116130 * cb + 32768) >> 16)
    return np.clip(np.stack([b, g, r], axis=-1), 0, 255).astype(np.uint8), info


# ---- the synchronisation ---------------------------------------------------------------------------------------------
INVALID = None


def sync_model(f, sub_bits=SUB_BITS, hops=SYNC_HOPS, per_read=SYNC_LAUNCHES_PER_READ):
    """The device's synchronisation of subsequence entry states for the file f.  Every restart segment is cut into
    subsequences of sub_bits bits; entry states (bit, block of the MCU, zig-zag index) start as guesses (first bit, 0, 0)
    and each launch lets every subsequence's decoder carry its state into up to `hops` following subsequences, as
    jdec_sync_kernel does.  In this model a decoder sees the states recorded at the launch's start for its own entry,
    and where two decoders record a state at the same boundary the one that started earlier in the segment wins (a
    launch in which no thread sees what lower threads record: the schedule that progresses least).  Returns a dict:
      subs            number of subsequences, per segment
      true            the true entry state of every subsequence
      guess_meets     per subsequence that is neither its segment's first (whose entry state is known) nor its last:
                      the decode from its guessed state reaches the true state of the next one (None for the others)
      guess_invalid   ... meets a code no table holds (or a run past 63) before the next one
      launches        launches until one changes nothing (that one included); rounds: host rounds of per_read launches
      invalid_marks   times an invalid state was recorded"""
    F = Frame(f)
    subs = []   # (begin, last, segment)
    per_seg = []
    for s in range(len(F.seg_bytes) - 1):
        b, e = F.seg_bytes[s], F.seg_bytes[s + 1]
        ns = max(1, (8 * (e - b) + sub_bits - 1) // sub_bits)
        per_seg.append(ns)
        for q in range(ns):
            subs.append((8 * b + q * sub_bits, q + 1 == ns, s))
    n = len(subs)
    memo = {}

    def advance(state, t):
        key = (state, t)
        if key in memo:
            return memo[key]
        pos, j, k = state
        if j >= F.bpm or k > 63:
            j = k = 0
        stop = subs[t][0]
        res = None
        while pos < stop:
            r = F.step(pos, j, k)
            if r is None:
                break
            pos, j, k = r[:3]
        else:
            res = (pos, j, k)
        memo[key] = res
        return res

    true = [None] * n
    for i in range(n):
        true[i] = (subs[i][0], 0, 0) if i == 0 or subs[i - 1][1] else advance(true[i - 1], i)
    guesses = [(subs[i][0], 0, 0) for i in range(n)]
    guessed = [i > 0 and not subs[i - 1][1] and not subs[i][1] for i in range(n)]
    meets = [advance(guesses[i], i + 1) == true[i + 1] if guessed[i] else None for i in range(n)]
    invalid = [advance(guesses[i], i + 1) is INVALID if guessed[i] else None for i in range(n)]
    entry = list(guesses)
    launches, marks = 0, 0
    while True:
        launches += 1
        changes = 0
        for i in reversed(range(n)):
            if subs[i][1]:
                continue
            st, t = entry[i], i + 1
            if st is INVALID:
                if entry[t] is not INVALID:
                    entry[t] = INVALID
                    changes += 1
                    marks += 1
                continue
            for _ in range(hops):
                now = advance(st, t)
                if entry[t] == now:
                    break
                entry[t] = now
                changes += 1
                marks += now is INVALID
                if now is INVALID or subs[t][1]:
                    break
                st, t = now, t + 1
        if changes == 0:
            break
    assert entry == true
    return dict(subs=per_seg, true=true, guess_meets=meets, guess_invalid=invalid, launches=launches,
                rounds=(launches + per_read - 1) // per_read, invalid_marks=marks)


# ---- the case set ---------------------------------------------------------------------------------------------------
def _flat_q(v):
    return np.full(64, v, np.int64)


def _gray(blocks, bx, q, dc=None, ac=None, stored_dc=True, **kw):
    """A gray file of the blocks (n, 64) laid out bx blocks wide.  stored_dc: element 0 of each block is the int16 value
    to store (the predictor values are derived per restart segment), else the predictor value written."""
    blocks = np.array(blocks, np.int64)
    if stored_dc:
        ri = kw.get("restart") or len(blocks)
        blocks[:, 0] = np.concatenate([_predictor(blocks[s:s + ri, 0]) for s in range(0, len(blocks), ri)])
    by = len(blocks) // bx
    assert by * bx == len(blocks)
    d, a = standard_tables()
    return write([blocks.reshape(by, bx, 64)], 8 * bx, 8 * by, "gray", [q], [dc or d], [ac or a], **kw)


def _lanes(rng, kind, n):
    """(blocks, q): n blocks aimed at one of the IDCT's 16-bit wraps or saturations, with quantisers."""
    b = np.zeros((n, 64), np.int64)
    q = _flat_q(1)
    if kind == "deq_wrap":        # dequantised products past int16
        q = rng.integers(2, 65536, 64)
        m = rng.random((n, 64)) < 0.3
        b[m] = rng.integers(-32767, 32768, m.sum())
    elif kind == "deq_edges":     # products exactly 32767 and -32768, nothing wrapping
        q = np.where(np.arange(64) % 2 == 0, 1, 2)
        for i in range(n):
            at = rng.choice(64, 6, replace=False)
            b[i, at] = np.where(at % 2 == 0, 32767, -16384)
    elif kind == "even_wrap":     # in0 + in4 / in0 - in4 past int16 (rows 0 and 4 of a column)
        for i in range(n):
            col = rng.integers(0, 8, 3)
            s = rng.choice([-1, 1])
            b[i, col] = s * rng.integers(16384, 32768, 3)
            b[i, 32 + col] = rng.choice([-1, 1]) * rng.integers(16384, 32768, 3)
    elif kind == "odd_wrap":      # in7 + in3, in5 + in1 past int16
        for i in range(n):
            col = rng.integers(0, 8, 2)
            s = rng.choice([-1, 1])
            b[i, 8 * 7 + col] = s * rng.integers(16384, 32768, 2)
            b[i, 8 * 3 + col] = s * rng.integers(16384, 32768, 2)
            b[i, 8 * 5 + col] = -s * rng.integers(16384, 32768, 2)
            b[i, 8 * 1 + col] = -s * rng.integers(16384, 32768, 2)
    elif kind == "pass1_sat":     # pass-1 sums past int16 without any 16-bit wrap before them
        for i in range(n):
            col = rng.integers(0, 8)
            b[i, col + 8 * np.arange(8)] = rng.choice([-1, 1]) * rng.integers(6000, 16000, 8) * [1, 1, 1, 0, 0, 0, 0, 0]
    elif kind == "shortcut":      # rows 1..7 zero, row-0 AC terms: DC * q fits in 16 bits, DC * q * 4 does not
        q = rng.integers(1, 20, 64)
        q[0] = 4
        for i in range(n):
            b[i, 0] = rng.choice([-1, 1]) * rng.integers(2048, 8192)
            b[i, 1:8] = np.where(rng.random(7) < 0.5, rng.integers(-1700, 1700, 7), 0)
            b[i, 1 + rng.integers(0, 7)] = rng.choice([-1, 1]) * rng.integers(1, 1700)
    elif kind == "clamp":         # outputs past both ends, nothing wrapping
        q = _flat_q(4)
        for i in range(n):
            b[i, 0] = rng.choice([-1, 1]) * rng.integers(300, 700)
            b[i, rng.integers(1, 64, 4)] = rng.integers(-200, 200, 4)
    return b, q


def _dc_values(diffs):
    return np.cumsum(np.asarray(diffs, np.int64))


def _predictor(stored):
    """DC predictor values whose int16 images are `stored` (but for a difference of 32768, which no category holds: that
    value is one less) and whose differences lie in [-32767, 32767]."""
    out, p = [], 0
    for v in np.asarray(stored, np.int64):
        d = wrap16(int(v) - p)
        p += d if d != -32768 else -32767
        out.append(p)
    return np.array(out, np.int64)


def cases():
    """[(name, file)]: the extreme-coefficient files every test of this set uses (tests/golden/jpeg_extreme_cases.npz
    holds them with cv2.imread's decodes)."""
    rng = np.random.default_rng(2026)
    out = []
    # IDCT lanes: each wrap or saturation in blocks of its own, gray, 8 x 12 blocks
    for kind in ("deq_wrap", "deq_edges", "even_wrap", "odd_wrap", "pass1_sat", "shortcut", "clamp"):
        for k in range(3):
            b, q = _lanes(rng, kind, 96)
            out.append(("lanes_%s_%d" % (kind, k), _gray(b, 8, q, restart=(0, 5, 1)[k])))
    # entropy: DC categories 12..15 and AC categories 11..15 (a predictor that wanders within int16)
    for k in range(2):
        n = 48
        b = np.zeros((n, 64), np.int64)
        dcd = rng.choice([-1, 1], n) * (1 << rng.integers(11, 15, n)) + rng.integers(0, 2048, n)
        m = rng.random((n, 64)) < 0.15
        b[m] = rng.choice([-1, 1], m.sum()) * rng.integers(1024, 32768, m.sum())
        b[:, 0] = np.clip(_dc_values(dcd), -30000, 30000)
        out.append(("categories_%d" % k, _gray(b, 8, _flat_q(1 + 7 * k), stored_dc=False, restart=4 * k)))
    # runs ending exactly at k = 63: a value at 63 after a run, trailing ZRLs to 64, EOB read at k = 63
    b = np.zeros((24, 64), np.int64)
    for i in range(24):
        zz = np.zeros(64, np.int64)
        zz[0] = rng.integers(-500, 500)
        if i % 3 == 0:
            zz[[5, 47, 63]] = rng.integers(1, 900, 3)          # run 15 into k = 63
        elif i % 3 == 1:
            zz[[3, 47]] = rng.integers(-900, -1, 2)            # 16 zeros left: one ZRL to 64
        else:
            zz[[31, 62]] = rng.integers(1, 900, 2)             # EOB at k = 63
        b[i, NATURAL] = zz
    out.append(("k63_eob", _gray(b, 6, _flat_q(3))))
    out.append(("k63_zrl_tail", _gray(b, 6, _flat_q(3), zrl_tail=True)))
    # 16-bit codes: a 256-symbol AC table and a DC table whose used symbols have 16-bit codes
    used_ac = [EOB, ZRL, 0x01, 0x0F, 0xF1, 0xFF, 0x1B, 0x3E]
    extra = [(r << 4) for r in range(1, 15)]                  # (r, 0), r < 15: EOB to libjpeg
    ac_all = [s for s in ac_symbols() if s not in used_ac] + extra
    ac16 = Huff.flat(ac_all, 8, used_ac, 16)
    assert len(ac16.vals) == 256
    dc16 = Huff([(s, 4) for s in range(2, 14)] + [(s, 16) for s in (0, 1, 14, 15)])
    b = np.zeros((40, 64), np.int64)
    for i in range(40):
        zz = np.zeros(64, np.int64)
        zz[0] = rng.choice([-1, 1]) * rng.integers(8192, 32767) if i % 2 else rng.integers(-1, 2)
        zz[1] = rng.choice([-1, 1])
        zz[2] = rng.choice([-1, 1]) * rng.integers(16384, 32768)
        zz[18] = rng.choice([-1, 1])                           # run 15, category 1
        zz[34] = rng.choice([-1, 1]) * rng.integers(16384, 32768)   # run 15, category 15
        zz[36] = rng.choice([-1, 1]) * rng.integers(1024, 2048)     # run 1, category 11
        zz[40] = rng.choice([-1, 1]) * rng.integers(8192, 16384)    # run 3, category 14
        b[i, NATURAL] = zz
    out.append(("long_codes", _gray(b, 8, _flat_q(5), dc=dc16, ac=ac16)))
    # a DC predictor past +-32767 inside one segment and across subsequence boundaries, reset at every restart
    for k, ri in enumerate((0, 48)):
        n = 192
        b = np.zeros((n, 64), np.int64)
        m = rng.random((n, 64)) < 0.5
        b[m] = rng.integers(-255, 256, m.sum())
        steps = np.where((np.arange(n) // 40) % 2 == 0, 1, -1) * rng.integers(20000, 32768, n)
        b[:, 0] = _dc_values(steps) if not ri else np.concatenate(
            [_dc_values(steps[s:s + ri]) for s in range(0, n, ri)])
        out.append(("dc_drift_%d" % k, _gray(b, 16, _flat_q(1 + k), stored_dc=False, restart=ri)))
    # colour: extreme chroma under Y = 0 and Y = 255, every sampling, MCU-remainder sizes
    for sampling in ("444", "422", "420"):
        for w, h in ((1, 1), (3, 5), (17, 9), (33, 18), (15, 31)):
            shapes = plane_shapes(w, h, sampling)
            planes = []
            for c, s in enumerate(shapes):
                p = np.zeros(s + (64,), np.int64)
                if c == 0:
                    p[..., 0] = rng.choice([-1024, 1024], s)
                else:
                    p[..., 0] = rng.choice([-1024, 1024, -700, 700], s)
                    m = rng.random(s + (64,)) < 0.2
                    m[..., 0] = False
                    p[m] = rng.integers(-3000, 3000, m.sum())
                planes.append(p)
            d, a = standard_tables()
            out.append(("colour_%s_%dx%d" % (sampling, w, h),
                        write(planes, w, h, sampling, [_flat_q(1), _flat_q(2), _flat_q(3)], [d] * 3, [a] * 3,
                              restart=(w * h) % 3)))
    out += sync_cases()
    return out


def _unit_tables(cat, eob_bits=16):
    """DC and AC tables of one 8-bit code each (category cat, and (0, cat)), the AC table with an EOB of eob_bits."""
    return Huff([(cat, 8)]), Huff([(cat, 8), (EOB, eob_bits)])


def sync_cases():
    """[(name, file)] for the synchronisation: see the tests in tests/test_gpu_jpeg_decode_extreme.py."""
    rng = np.random.default_rng(7)
    out = []
    # Every codeword is 16 bits (an 8-bit code and 8 value bits): subsequence boundaries (multiples of 8192 bits) fall
    # on codeword boundaries, and a guess (block start) is true only where a block starts.  A first block of 37
    # codewords (EOB at k = 36) and 64-codeword blocks after it put every boundary at k = 27: the decodes from guesses
    # keep their offset of 27 coefficients and never meet the true states.  2176 blocks: 272 subsequences in one segment.
    dct, act = _unit_tables(8)
    n = 2176
    pattern = np.where(np.arange(64) % 3 == 0, 200, -140)
    b = np.tile(pattern, (n, 1))
    b[0, [NATURAL[k] for k in range(36, 64)]] = 0
    b[:, 0] = 150 * np.arange(1, n + 1)   # a predictor far past int16
    out.append(("sync_never", _gray(b, 64, _flat_q(1), dc=dct, ac=act, stored_dc=False)))
    # 9-bit codewords (8-bit code 0x00, one value bit): a guess that starts inside a codeword soon reads 0x01, a code
    # neither table holds
    dct, act = _unit_tables(1)
    n = 448
    b = rng.choice([-1, 1], (n, 64))
    b[:, 0] = _dc_values(b[:, 0])
    out.append(("sync_invalid", _gray(b, 32, _flat_q(1), dc=dct, ac=act, stored_dc=False)))
    # 1024-bit blocks: restart segments of exactly 1, 2 and 3 subsequences, and shorter than one
    dct, act = _unit_tables(8)
    b = np.tile(pattern, (96, 1)) * np.where(rng.random((96, 1)) < 0.5, 1, -1)
    for ri in (1, 3, 8, 16, 24):
        c = b.copy()
        c[:, 0] = np.concatenate([_dc_values(np.full(min(ri, 96 - s), 170)) for s in range(0, 96, ri)])
        out.append(("segments_ri%d" % ri, _gray(c, 12, _flat_q(1), dc=dct, ac=act, stored_dc=False, restart=ri)))
    return out


def ortho_frames(n, width, height, colored, seed=0):
    """n camera frames of extreme content (4:2:0 colour or gray, width x height): sparse coefficients of every
    magnitude under wide quantisers, a restart interval of 3 MCUs."""
    rng = np.random.default_rng(seed)
    sampling = "420" if colored else "gray"
    dc, ac = standard_tables()
    out = []
    for _ in range(n):
        planes = []
        for s in plane_shapes(width, height, sampling):
            p = np.zeros(s + (64,), np.int64)
            m = rng.random(s + (64,)) < 0.06
            p[m] = rng.choice([-1, 1], m.sum()) * (1 << rng.integers(0, 15, m.sum()))
            p[..., 0] = rng.integers(-16000, 16000, s)
            planes.append(p)
        q = [rng.integers(1, 300, 64) for _ in planes]
        out.append(write(planes, width, height, sampling, q, [dc] * len(planes), [ac] * len(planes), restart=3))
    return out
