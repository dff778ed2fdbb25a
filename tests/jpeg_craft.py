"""JPEG files for the decoder tests: cv2.imencode variants (sampling, quality, restart interval, optimised tables), edits
of their marker segments (DHT removed, an EXIF orientation inserted, patched markers), and a small baseline writer for
what cv2's encoder cannot reach: chosen quantised coefficient blocks, quantisation tables and sampling, entropy-coded
with the standard tables of T.81 Annex K.3 (written out, or left for the decoder to supply as MJPEG frames do)."""
import struct

import numpy as np

SAMPLINGS = ("444", "422", "440", "420", "411", "gray")
# luma (h, v) of each cv2 sampling
LUMA = {"444": (1, 1), "422": (2, 1), "440": (1, 2), "420": (2, 2), "411": (4, 1)}


def encode(img, sampling="420", quality=90, restart=0, optimize=False, progressive=False):
    """cv2.imencode of a BGR frame (or its gray conversion for sampling "gray") -> bytes."""
    import cv2
    params = [cv2.IMWRITE_JPEG_QUALITY, int(quality), cv2.IMWRITE_JPEG_RST_INTERVAL, int(restart),
              cv2.IMWRITE_JPEG_OPTIMIZE, int(optimize), cv2.IMWRITE_JPEG_PROGRESSIVE, int(progressive)]
    if sampling == "gray":
        img = cv2.cvtColor(img, cv2.COLOR_BGR2GRAY) if img.ndim == 3 else img
    else:
        params += [cv2.IMWRITE_JPEG_SAMPLING_FACTOR, getattr(cv2, "IMWRITE_JPEG_SAMPLING_FACTOR_" + sampling)]
    ok, buf = cv2.imencode(".jpg", img, params)
    assert ok
    return buf.tobytes()


def decode(data):
    """cv2.imdecode(bytes, IMREAD_COLOR): the decoder's reference."""
    import cv2
    return cv2.imdecode(np.frombuffer(data, np.uint8), cv2.IMREAD_COLOR)


def markers(data):
    """[(marker, start, end)] of the segments before the scan data (start at 0xFF, end after the payload); SOS last."""
    out, i = [], 2
    while i < len(data):
        m = data[i + 1]
        n = struct.unpack(">H", data[i + 2:i + 4])[0]
        out.append((m, i, i + 2 + n))
        if m == 0xDA:
            break
        i += 2 + n
    return out


def strip(data, marker):
    """The file without its segments of one marker (e.g. 0xC4: no DHT, as an MJPEG frame)."""
    cut = [(a, b) for m, a, b in markers(data) if m == marker]
    out, last = bytearray(), 0
    for a, b in cut:
        out += data[last:a]
        last = b
    return bytes(out + data[last:])


def insert(data, segment, after=0xE0):
    """A marker segment (bytes from 0xFF) inserted after the last segment of marker `after` (or after SOI)."""
    pos = 2
    for m, a, b in markers(data):
        if m == after:
            pos = b
    return data[:pos] + segment + data[pos:]


def app_segment(marker, payload):
    return bytes([0xFF, marker]) + struct.pack(">H", len(payload) + 2) + payload


def exif(orientation, big_endian=False):
    """An APP1 Exif segment whose IFD0 holds the Orientation tag (0x0112, SHORT) and one other tag."""
    e = ">" if big_endian else "<"
    tiff = (b"MM" if big_endian else b"II") + struct.pack(e + "HI", 42, 8)
    entries = [struct.pack(e + "HHI", 0x010F, 2, 4) + b"cam\0",                       # Make, inline ASCII
               struct.pack(e + "HHIH", 0x0112, 3, 1, orientation) + b"\0\0"]
    ifd = struct.pack(e + "H", len(entries)) + b"".join(entries) + struct.pack(e + "I", 0)
    return app_segment(0xE1, b"Exif\0\0" + tiff + ifd)


def with_orientation(data, orientation, big_endian=False):
    return insert(data, exif(orientation, big_endian))


def patch_marker(data, old, new):
    """The first segment of marker `old` re-labelled as `new` (e.g. SOF0 -> SOF9)."""
    for m, a, b in markers(data):
        if m == old:
            return data[:a + 1] + bytes([new]) + data[a + 2:]
    raise ValueError("no marker %#x" % old)


def scan_range(data):
    """(begin, end) of the entropy-coded data: after the SOS segment, to the EOI."""
    sos = markers(data)[-1]
    assert sos[0] == 0xDA and data[-2:] == b"\xff\xd9"
    return sos[2], len(data) - 2


# ---------------------------------------------------------------- the baseline writer
# T.81 Annex K.3: bits[l - 1] = codes of length l, then the symbols; tables 0 (luma) and 1 (chroma)
STD_DC_BITS = [[0, 1, 5, 1, 1, 1, 1, 1, 1, 0, 0, 0, 0, 0, 0, 0], [0, 3, 1, 1, 1, 1, 1, 1, 1, 1, 1, 0, 0, 0, 0, 0]]
STD_AC_BITS = [[0, 2, 1, 3, 3, 2, 4, 3, 5, 5, 4, 4, 0, 0, 1, 0x7d], [0, 2, 1, 2, 4, 4, 3, 4, 7, 5, 4, 4, 0, 1, 2, 0x77]]


def std_ac_vals(t):
    """The 162 AC symbols of K.5 (t = 0) / K.6 (t = 1), as cv2 writes them: read from a cv2-encoded file."""
    for m, a, b in markers(encode(np.zeros((8, 8, 3), np.uint8), "444", 75)):
        if m != 0xC4:
            continue
        seg = memoryview(encode(np.zeros((8, 8, 3), np.uint8), "444", 75))[a + 4:b]
        i = 0
        while i < len(seg):
            tc, th = seg[i] >> 4, seg[i] & 15
            bits = list(seg[i + 1:i + 17])
            n = sum(bits)
            if tc == 1 and th == t:
                return bytes(seg[i + 17:i + 17 + n])
            i += 17 + n
    raise AssertionError("no standard AC table")


def dht_tables(data):
    """{(class, id): (bits[16], symbols)} of every DHT segment of a file."""
    out = {}
    for m, a, b in markers(data):
        if m != 0xC4:
            continue
        seg = data[a + 4:b]
        i = 0
        while i < len(seg):
            bits = list(seg[i + 1:i + 17])
            n = sum(bits)
            out[(seg[i] >> 4, seg[i] & 15)] = (bits, bytes(seg[i + 17:i + 17 + n]))
            i += 17 + n
    return out


def _codes(bits, vals):
    """Canonical Huffman codes (T.81 Annex C): symbol -> (code, length)."""
    out, code, k = {}, 0, 0
    for l in range(1, 17):
        for _ in range(bits[l - 1]):
            out[vals[k]] = (code, l)
            code += 1
            k += 1
        code <<= 1
    return out


class _Bits:
    def __init__(self):
        self.acc, self.n, self.out = 0, 0, bytearray()

    def put(self, v, n):
        for i in range(n - 1, -1, -1):
            self.acc = (self.acc << 1) | ((v >> i) & 1)
            self.n += 1
            if self.n == 8:
                self.out.append(self.acc)
                if self.acc == 0xFF:
                    self.out.append(0)
                self.acc, self.n = 0, 0

    def flush(self):
        if self.n:
            self.put((1 << (8 - self.n)) - 1, 8 - self.n)


def _size(v):
    return 0 if v == 0 else int(abs(int(v))).bit_length()


def _extra(v, s):
    return v if v >= 0 else v + (1 << s) - 1


ZIGZAG = [0, 1, 8, 16, 9, 2, 3, 10, 17, 24, 32, 25, 18, 11, 4, 5, 12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13, 6, 7, 14,
          21, 28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53, 60,
          61, 54, 47, 55, 62, 63]


def write(width, height, blocks, quant, luma=(1, 1), gray=False, restart=0, dht=True, qbits=8, app0=True):
    """A baseline JPEG of quantised coefficient blocks.  blocks: int [nblocks, 64] in decode order (MCU by MCU, each
    MCU its luma blocks row by row then Cb, Cr), natural order, DC as values (not differences).  quant: [ncomp][64]
    natural order (luma table, then one chroma table for both chroma components).  dht=False leaves the standard
    tables to the decoder."""
    nc = 1 if gray else 3
    h0, v0 = (1, 1) if gray else luma
    mcux, mcuy = -(-width // (8 * h0)), -(-height // (8 * v0))
    bpm = 1 if gray else h0 * v0 + 2
    assert len(blocks) == mcux * mcuy * bpm
    out = bytearray(b"\xff\xd8")
    if app0:
        out += app_segment(0xE0, b"JFIF\0\x01\x01\0\0\x01\0\x01\0\0")
    for t, q in enumerate(quant[:min(nc, 2)]):
        q = np.asarray(q).reshape(-1)
        if qbits == 8:
            body = bytes([t]) + bytes(int(q[ZIGZAG[k]]) for k in range(64))
        else:
            body = bytes([0x10 | t]) + b"".join(struct.pack(">H", int(q[ZIGZAG[k]])) for k in range(64))
        out += app_segment(0xDB, body)
    comps = [(1, (h0 << 4) | v0, 0)] + ([] if gray else [(2, 0x11, 1), (3, 0x11, 1)])
    out += app_segment(0xC0, bytes([8]) + struct.pack(">HH", height, width) + bytes([nc]) +
                       b"".join(bytes(c) for c in comps))
    ac_vals = [std_ac_vals(0), std_ac_vals(1)]
    dc_vals = [bytes(range(12))] * 2
    if dht:
        for t in range(1 if gray else 2):
            out += app_segment(0xC4, bytes([t]) + bytes(STD_DC_BITS[t]) + dc_vals[t])
            out += app_segment(0xC4, bytes([0x10 | t]) + bytes(STD_AC_BITS[t]) + ac_vals[t])
    if restart:
        out += app_segment(0xDD, struct.pack(">H", restart))
    out += app_segment(0xDA, bytes([nc]) + b"".join(bytes([c[0], (c[2] << 4) | c[2]]) for c in comps) + b"\x00\x3f\x00")
    dc_codes = [_codes(STD_DC_BITS[t], dc_vals[t]) for t in range(2)]
    ac_codes = [_codes(STD_AC_BITS[t], ac_vals[t]) for t in range(2)]
    bw = _Bits()
    pred = [0, 0, 0]
    nmcu = mcux * mcuy
    for m in range(nmcu):
        if restart and m and m % restart == 0:
            bw.flush()
            out += bw.out
            out += bytes([0xFF, 0xD0 + ((m // restart - 1) & 7)])
            bw, pred = _Bits(), [0, 0, 0]
        for r in range(bpm):
            c = 0 if gray or r < h0 * v0 else 1 + r - h0 * v0
            t = 0 if c == 0 else 1
            blk = np.asarray(blocks[m * bpm + r]).reshape(-1)
            diff = int(blk[0]) - pred[c]
            pred[c] = int(blk[0])
            s = _size(diff)
            bw.put(*dc_codes[t][s])
            if s:
                bw.put(_extra(diff, s), s)
            run = 0
            for k in range(1, 64):
                v = int(blk[ZIGZAG[k]])
                if v == 0:
                    run += 1
                    continue
                while run > 15:
                    bw.put(*ac_codes[t][0xF0])
                    run -= 16
                s = _size(v)
                bw.put(*ac_codes[t][(run << 4) | s])
                bw.put(_extra(v, s), s)
                run = 0
            if run:
                bw.put(*ac_codes[t][0x00])
    bw.flush()
    out += bw.out + b"\xff\xd9"
    return bytes(out)
