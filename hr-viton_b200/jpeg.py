"""Baseline JPEG decoding on the GPU, bit-identical to PIL (libjpeg-turbo's default decode: islow IDCT, fancy upsampling, separate
upsample-then-convert colour path).

parse() reads a file's markers on the host into a Header: size, components and sampling, quantisation tables, Huffman tables as
BITS/HUFFVAL, the restart interval, and the byte range of the entropy-coded segment with the offsets of its RSTn markers.
device_decodable(header) is the one place that decides which files the device decodes; every other file stays on PIL.  decode()
runs a batch of files through the three kernels of include/hrviton_sm100_jpeg.h (one launch per stage for the whole batch, whatever
the images' sizes, samplings and component counts); decode_np() is the same decoder in numpy, the CPU oracle the tests hold against
PIL.

Device-decodable: 8-bit baseline / extended-sequential Huffman (SOF0 / SOF1), one scan holding every component, the colour space
libjpeg infers is grayscale (one component) or YCbCr (three), and luma sampling 1x1, 2x1 or 2x2 with chroma 1x1 (4:4:4, 4:2:2,
4:2:0).  Progressive, arithmetic, 12-bit, CMYK / YCCK, RGB-coded, multi-scan and other samplings go to PIL."""
import ctypes

import numpy as np
import torch

from . import capi

SOI, EOI, SOS, DQT, DHT, DRI = 0xD8, 0xD9, 0xDA, 0xDB, 0xC4, 0xDD
SOF_HUFFMAN_SEQUENTIAL = (0xC0, 0xC1)
SOF_ALL = (0xC0, 0xC1, 0xC2, 0xC3, 0xC5, 0xC6, 0xC7, 0xC9, 0xCA, 0xCB, 0xCD, 0xCE, 0xCF)

# natural index of each zig-zag position, padded with 63 as libjpeg's jpeg_natural_order is: a corrupt run past coefficient 63
# lands on 63 instead of outside the block
ZIGZAG = np.array([0, 1, 8, 16, 9, 2, 3, 10, 17, 24, 32, 25, 18, 11, 4, 5, 12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13, 6, 7, 14, 21, 28,
                   35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55,
                   62, 63] + [63] * 16, np.int32)

ERR_BAD_CODE, ERR_TRUNCATED = 1, 2  # per-image error codes of hrv_jpeg_huffman
_ERRORS = {ERR_BAD_CODE: "corrupt entropy-coded data (a Huffman code with no table entry)",
           ERR_TRUNCATED: "the entropy-coded segment ends before the last block (image file is truncated)"}


class Header:
    """What parse() reads from one file.  Offsets are file offsets; `segment` is [start, end) of the scan's entropy-coded data and
    `rst` the offsets of its RSTn markers."""

    def __init__(self):
        self.sof = None
        self.precision = 8
        self.height = self.width = 0
        self.components = []  # (id, h, v, quant table id) in frame order
        self.quant = {}  # table id -> uint16 [64], natural order
        self.huffman = {}  # (0 = DC / 1 = AC, id) -> (BITS uint8 [16], HUFFVAL uint8 [n])
        self.restart_interval = 0
        self.scans = []  # (component ids, DC table ids, AC table ids, Ss, Se, Ah, Al)
        self.scan_tables = None  # tables in force at the first scan: quant, huffman
        self.segment = (0, 0)
        self.rst = np.zeros(0, np.int64)
        self.jfif = False
        self.adobe_transform = None

    @property
    def mode(self):
        """PIL's mode for the file: its component count decides."""
        return {1: "L", 3: "RGB", 4: "CMYK"}.get(len(self.components))

    @property
    def size(self):
        return self.width, self.height

    @property
    def layer(self):
        """PIL's JpegImageFile.layer: (id, h, v, quant table id) per component (PIL's comment names the middle two the other way)."""
        return list(self.components)

    @property
    def quantization(self):
        """PIL's JpegImageFile.quantization: {table id: 64 values in natural order}."""
        return {k: [int(x) for x in v] for k, v in self.quant.items()}

    def color_space(self):
        """The colour space libjpeg infers (jdapimin.c default_decompress_parms): 'GRAYSCALE', 'YCbCr', 'RGB', 'CMYK', 'YCCK' or None."""
        n = len(self.components)
        if n == 1:
            return "GRAYSCALE"
        if n == 3:
            if self.jfif:
                return "YCbCr"
            if self.adobe_transform is not None:
                return "RGB" if self.adobe_transform == 0 else "YCbCr"
            ids = tuple(c[0] for c in self.components)
            return "RGB" if ids == (82, 71, 66) else "YCbCr"
        if n == 4:
            if self.adobe_transform is not None:
                return "YCCK" if self.adobe_transform == 2 else "CMYK"
            return "CMYK"
        return None


def _u16(d, i):
    return (int(d[i]) << 8) | int(d[i + 1])


def _check_huffman(bits, vals):
    """libjpeg's jpeg_make_d_derived_tbl checks: no more than 256 symbols, and no code overflows its length."""
    if int(bits.sum()) > 256 or len(vals) < int(bits.sum()):
        raise SyntaxError("bad Huffman table")
    code = 0
    for l in range(16):
        code += int(bits[l])
        if code > (1 << (l + 1)):
            raise SyntaxError("bad Huffman table")
        code <<= 1


def _segment_end(a, start):
    """(end of the entropy-coded data starting at `start`, offsets of its RSTn markers): the first 0xFF not followed by a stuffed
    0x00, an RSTn or a fill byte ends it.  numpy over the bytes, no Python loop."""
    tail = a[start:]
    ff = np.flatnonzero(tail[:-1] == 0xFF)
    nxt = tail[ff + 1]
    rst = ff[(nxt >= 0xD0) & (nxt <= 0xD7)]
    end = ff[(nxt != 0x00) & ((nxt < 0xD0) | (nxt > 0xD7)) & (nxt != 0xFF)]
    if len(end) == 0:
        raise OSError("image file is truncated (no marker after the entropy-coded segment)")
    e = int(end[0])
    fills = ff[(nxt == 0xFF) & (ff < e)]  # fill bytes (0xFF 0xFF ...) before the marker belong to the marker
    while len(fills) and int(fills[-1]) == e - 1:
        e -= 1
        fills = fills[:-1]
    return start + e, start + rst[rst < e].astype(np.int64)


def parse(data):
    """Header of the JPEG file `data` (bytes or a path).  Raises SyntaxError on data that is not a JPEG file or has bad tables, and
    OSError('image file is truncated ...') on a file cut before its EOI, as PIL does on loading it."""
    if isinstance(data, str):
        with open(data, "rb") as f:
            data = f.read()
    a = np.frombuffer(data, np.uint8)
    if len(a) < 4 or a[0] != 0xFF or a[1] != SOI:
        raise SyntaxError("not a JPEG file")
    h = Header()
    i = 2
    n = len(a)
    while True:
        while i < n and a[i] == 0xFF and i + 1 < n and a[i + 1] == 0xFF:  # fill bytes
            i += 1
        if i + 1 >= n:
            raise OSError("image file is truncated (no EOI marker)")
        if a[i] != 0xFF:
            raise SyntaxError("no marker at offset %d" % i)
        m = int(a[i + 1])
        i += 2
        if m == EOI:
            break
        if 0xD0 <= m <= 0xD7 or m == 0x01:
            continue
        if i + 2 > n:
            raise OSError("image file is truncated (in a marker)")
        length = _u16(a, i)
        if length < 2 or i + length > n:
            raise OSError("image file is truncated (in marker 0x%02X)" % m)
        s = a[i + 2:i + length]
        i += length
        if m == 0xE0 and len(s) >= 14 and bytes(s[:5]) == b"JFIF\0":
            h.jfif = True
        elif m == 0xEE and len(s) >= 12 and bytes(s[:5]) == b"Adobe":
            h.adobe_transform = int(s[11])
        elif m == DQT:
            j = 0
            while j < len(s):
                pq, tq = int(s[j]) >> 4, int(s[j]) & 15
                size = 64 * (2 if pq else 1)
                if j + 1 + size > len(s) or tq > 3:
                    raise SyntaxError("bad quantization table marker")
                v = s[j + 1:j + 1 + size]
                zz = (v[0::2].astype(np.uint16) << 8 | v[1::2]) if pq else v.astype(np.uint16)
                q = np.zeros(64, np.uint16)
                q[ZIGZAG[:64]] = zz
                h.quant[tq] = q
                j += 1 + size
        elif m == DHT:
            j = 0
            while j < len(s):
                if j + 17 > len(s):
                    raise SyntaxError("bad Huffman table marker")
                tc, th = int(s[j]) >> 4, int(s[j]) & 15
                bits = s[j + 1:j + 17].copy()
                cnt = int(bits.sum())
                vals = s[j + 17:j + 17 + cnt].copy()
                _check_huffman(bits, vals)
                if tc > 1 or th > 3:
                    raise SyntaxError("bad Huffman table marker")
                h.huffman[(tc, th)] = (bits, vals)
                j += 17 + cnt
        elif m == DRI:
            if len(s) < 2:
                raise SyntaxError("bad DRI marker")
            h.restart_interval = _u16(s, 0)
        elif m in SOF_ALL:
            if h.sof is not None:
                raise SyntaxError("two frame headers")
            if len(s) < 6:
                raise SyntaxError("bad SOF marker")
            h.sof, h.precision = m, int(s[0])
            h.height, h.width = _u16(s, 1), _u16(s, 3)
            nc = int(s[5])
            if len(s) < 6 + 3 * nc:
                raise SyntaxError("bad SOF marker")
            h.components = [(int(s[6 + 3 * k]), int(s[7 + 3 * k]) >> 4, int(s[7 + 3 * k]) & 15, int(s[8 + 3 * k])) for k in range(nc)]
        elif m == SOS:
            if h.sof is None or len(s) < 1:
                raise SyntaxError("scan before the frame header")
            ns = int(s[0])
            if len(s) < 1 + 2 * ns + 3:
                raise SyntaxError("bad SOS marker")
            ids = tuple(int(s[1 + 2 * k]) for k in range(ns))
            td = tuple(int(s[2 + 2 * k]) >> 4 for k in range(ns))
            ta = tuple(int(s[2 + 2 * k]) & 15 for k in range(ns))
            ss, se, ahal = int(s[1 + 2 * ns]), int(s[2 + 2 * ns]), int(s[3 + 2 * ns])
            h.scans.append((ids, td, ta, ss, se, ahal >> 4, ahal & 15))
            end, rst = _segment_end(a, i)
            if len(h.scans) == 1:
                h.segment, h.rst = (i, end), rst
                h.scan_tables = ({k: v.copy() for k, v in h.quant.items()}, dict(h.huffman), h.restart_interval)
            i = end
    if h.sof is None or not h.scans:
        raise SyntaxError("no frame header or no scan")
    if h.width == 0 or h.height == 0:
        raise SyntaxError("image size 0 (a DNL marker is not supported)")
    return h


def _sampling(h):
    """(hmax, vmax) the device and decode_np use: the luma sampling of a three-component file, 1x1 for one component (a lone
    component is upsampled by nothing whatever its factors say)."""
    if len(h.components) == 1:
        return 1, 1
    return h.components[0][1], h.components[0][2]


def device_decodable(h):
    """True when the device decodes this file bit for bit as PIL does; every other file stays on PIL."""
    if h.sof not in SOF_HUFFMAN_SEQUENTIAL or h.precision != 8 or len(h.scans) != 1:
        return False
    nc = len(h.components)
    if h.color_space() not in ("GRAYSCALE", "YCbCr") or nc not in (1, 3):
        return False
    ids, td, ta, ss, se, ah, al = h.scans[0]
    if sorted(ids) != sorted(c[0] for c in h.components) or len(set(ids)) != nc or (ss, se, ah, al) != (0, 63, 0, 0):
        return False
    if ids != tuple(c[0] for c in h.components):  # libjpeg decodes in scan order; the device assumes frame order
        return False
    if nc == 3:
        samp = tuple((c[1], c[2]) for c in h.components)
        if samp[0] not in ((1, 1), (2, 1), (2, 2)) or samp[1] != (1, 1) or samp[2] != (1, 1):
            return False
    quant, huff, ri = h.scan_tables
    if any(c[3] not in quant for c in h.components):
        return False
    if any((0, t) not in huff for t in td) or any((1, t) not in huff for t in ta):
        return False
    # the restart markers must split the scan exactly as the restart interval says (libjpeg resynchronises otherwise)
    mx, my = _mcus(h)
    n_mcu = mx * my
    n_seg = (n_mcu + ri - 1) // ri if ri else 1
    return len(h.rst) == n_seg - 1


def _mcus(h):
    hm, vm = _sampling(h)
    return -(-h.width // (8 * hm)), -(-h.height // (8 * vm))


def _component_geometry(h):
    """Per component: (h samp, v samp, blocks per row, blocks per column) of the padded block grid, and its downsampled size
    (width, height) = ceil(image size * samp / max samp)."""
    hm, vm = _sampling(h)
    mx, my = _mcus(h)
    out = []
    for k in range(len(h.components)):
        hs, vs = (hm, vm) if k == 0 else (1, 1)
        out.append((hs, vs, mx * hs, my * vs, -(-h.width * hs // hm), -(-h.height * vs // vm)))
    return out


def entropy_segments(h):
    """[start, end) file offsets of each restart interval's data (the whole scan when there is no restart interval)."""
    starts = [h.segment[0]] + [int(r) + 2 for r in h.rst]
    ends = [int(r) for r in h.rst] + [h.segment[1]]
    return list(zip(starts, ends))


# ------------------------------------------------------------------------------------------------ numpy oracle

def _unstuff(b):
    """The segment's bytes with each stuffed 0x00 after 0xFF removed."""
    keep = np.ones(len(b), bool)
    ff = np.flatnonzero(b[:-1] == 0xFF)
    keep[ff[b[ff + 1] == 0x00] + 1] = False
    return b[keep]


def _lookup16(bits, vals):
    """(length, symbol) of every 16-bit lookahead: length 0 where no code matches."""
    length = np.zeros(1 << 16, np.int32)
    sym = np.zeros(1 << 16, np.int32)
    code, p = 0, 0
    for l in range(1, 17):
        for _ in range(int(bits[l - 1])):
            lo, hi = code << (16 - l), (code + 1) << (16 - l)
            length[lo:hi], sym[lo:hi] = l, int(vals[p])
            code += 1
            p += 1
        code <<= 1
    return length.tolist(), sym.tolist()


def _huffman_np(h, data):
    """Raw int16 coefficients, natural order, of every component: list of (blocks y, blocks x, 64)."""
    quant, huff, ri = h.scan_tables
    geo = _component_geometry(h)
    coefs = [np.zeros((g[3], g[2], 64), np.int16) for g in geo]
    _, td, ta = h.scans[0][:3]
    dc = [_lookup16(*huff[(0, t)]) for t in td]
    ac = [_lookup16(*huff[(1, t)]) for t in ta]
    mx, my = _mcus(h)
    n_mcu = mx * my
    per = ri if ri else n_mcu
    zz = ZIGZAG.tolist()
    a = np.frombuffer(data, np.uint8)
    for seg, (s0, s1) in enumerate(entropy_segments(h)):
        b = _unstuff(a[s0:s1])
        nbits = 8 * len(b)
        b = np.concatenate([b, np.zeros(8, np.uint8)]).astype(np.uint32)  # zeros past the end, as libjpeg feeds at a marker
        w32 = ((b[:-3] << 24) | (b[1:-2] << 16) | (b[2:-1] << 8) | b[3:]).tolist()
        pos = 0

        def bits(k):
            nonlocal pos
            if pos > nbits:
                raise ValueError(_ERRORS[ERR_TRUNCATED])
            v = (w32[pos >> 3] >> (32 - k - (pos & 7))) & ((1 << k) - 1)
            pos += k
            return v

        def decode(tab):
            nonlocal pos
            if pos > nbits:
                raise ValueError(_ERRORS[ERR_TRUNCATED])
            look = (w32[pos >> 3] >> (16 - (pos & 7))) & 0xFFFF
            l = tab[0][look]
            if l == 0:
                raise ValueError(_ERRORS[ERR_TRUNCATED if pos + 16 > nbits else ERR_BAD_CODE])
            pos += l
            return tab[1][look]

        def extend(s):
            v = bits(s)
            return v - (1 << s) + 1 if v < (1 << (s - 1)) else v

        pred = [0] * len(geo)
        for m in range(seg * per, min((seg + 1) * per, n_mcu)):
            mcx, mcy = m % mx, m // mx
            for c, (hs, vs, bw, bh, _, _) in enumerate(geo):
                for by in range(vs):
                    for bx in range(hs):
                        blk = coefs[c][mcy * vs + by, mcx * hs + bx]
                        s = decode(dc[c])
                        if s > 16:
                            raise ValueError(_ERRORS[ERR_BAD_CODE])
                        pred[c] += extend(s) if s else 0
                        blk[0] = np.int16(((pred[c] + 32768) & 0xFFFF) - 32768)
                        k = 1
                        while k < 64:
                            rs = decode(ac[c])
                            r, s = rs >> 4, rs & 15
                            if s:
                                k += r
                                blk[zz[k]] = extend(s)
                            elif r != 15:
                                break
                            else:
                                k += 15
                            k += 1
                        if pos > nbits:
                            raise ValueError(_ERRORS[ERR_TRUNCATED])
    return coefs


# libjpeg's jidctint.c constants: FIX(x) = round(x * 2^13)
CONST_BITS, PASS1_BITS = 13, 2
F_0_298, F_0_390, F_0_541, F_0_765, F_0_899, F_1_175 = 2446, 3196, 4433, 6270, 7373, 9633
F_1_501, F_1_847, F_1_961, F_2_053, F_2_562, F_3_072 = 12299, 15137, 16069, 16819, 20995, 25172


def _idct_1d(x, shift):
    """One islow pass over axis 1 of x (..., 8, ...) as int64, descaled by `shift` with rounding: jidctint.c's even / odd parts."""
    z2, z3 = x[:, 2], x[:, 6]
    z1 = (z2 + z3) * F_0_541
    tmp2 = z1 - z3 * F_1_847
    tmp3 = z1 + z2 * F_0_765
    tmp0 = (x[:, 0] + x[:, 4]) << CONST_BITS
    tmp1 = (x[:, 0] - x[:, 4]) << CONST_BITS
    t10, t13, t11, t12 = tmp0 + tmp3, tmp0 - tmp3, tmp1 + tmp2, tmp1 - tmp2
    o0, o1, o2, o3 = x[:, 7], x[:, 5], x[:, 3], x[:, 1]
    z1, z2, z3, z4 = o0 + o3, o1 + o2, o0 + o2, o1 + o3
    z5 = (z3 + z4) * F_1_175
    o0, o1, o2, o3 = o0 * F_0_298, o1 * F_2_053, o2 * F_3_072, o3 * F_1_501
    z1, z2, z3, z4 = z1 * -F_0_899, z2 * -F_2_562, z3 * -F_1_961 + z5, z4 * -F_0_390 + z5
    o0, o1, o2, o3 = o0 + z1 + z3, o1 + z2 + z4, o2 + z2 + z3, o3 + z1 + z4
    r = 1 << (shift - 1)
    return np.stack([t10 + o3, t11 + o2, t12 + o1, t13 + o0, t13 - o0, t12 - o1, t11 - o2, t10 - o3], 1) + r >> shift


def idct_islow_np(coefs, q):
    """libjpeg's jpeg_idct_islow of blocks (N, 64) raw int16 coefficients, natural order, with quantisation table q (64): uint8 (N, 8, 8).
    Columns first, then rows; the result is clamped to 0-255 (libjpeg-turbo's SIMD saturates; its C version masks a table index,
    which differs only for values a valid file does not produce)."""
    x = coefs.reshape(-1, 8, 8).astype(np.int64) * q.reshape(8, 8).astype(np.int64)
    ws = _idct_1d(x, CONST_BITS - PASS1_BITS)  # (N, 8 rows, 8 columns): axis 1 ran down each column
    out = _idct_1d(ws.transpose(0, 2, 1), CONST_BITS + PASS1_BITS + 3).transpose(0, 2, 1)
    return np.clip(out + 128, 0, 255).astype(np.uint8)


def upsample_np(p, cw, ch, hs, vs, w, h):
    """libjpeg-turbo's upsampling of a component (padded plane p, downsampled size cw x ch) to w x h: fancy (triangle) for h2v1 /
    h2v2 when the component is wider than 2 samples, replication otherwise.  Edges repeat the last real sample."""
    if (hs, vs) == (1, 1):
        return p[:h, :w]
    x = np.arange(w)
    y = np.arange(h)
    cx = x >> 1
    cy = y >> 1 if vs == 2 else y
    if cw <= 2:
        return p[cy][:, cx]
    p = p.astype(np.int32)
    odd = (x & 1).astype(np.int32)
    far_x = np.where(odd == 1, np.minimum(cx + 1, cw - 1), np.maximum(cx - 1, 0))
    if vs == 1:
        rows = p[y]
        return ((3 * rows[:, cx] + rows[:, far_x] + 1 + odd) >> 2).astype(np.uint8)
    far_y = np.where(y & 1, np.minimum(cy + 1, ch - 1), np.maximum(cy - 1, 0))
    colsum = 3 * p[cy] + p[far_y]  # (h, padded width)
    return ((3 * colsum[:, cx] + colsum[:, far_x] + 8 - odd) >> 4).astype(np.uint8)


def _fix16(v):
    return int(v * 65536 + 0.5)


C_R_CR, C_G_CB, C_G_CR, C_B_CB = _fix16(1.402), _fix16(0.34414), _fix16(0.71414), _fix16(1.772)


def ycc_to_rgb_np(y, cb, cr):
    y, cb, cr = (v.astype(np.int64) for v in (y, cb, cr))
    cb, cr = cb - 128, cr - 128
    r = y + ((C_R_CR * cr + 32768) >> 16)
    g = y + ((-C_G_CB * cb + 32768 - C_G_CR * cr) >> 16)
    b = y + ((C_B_CB * cb + 32768) >> 16)
    return np.clip(np.stack([r, g, b], -1), 0, 255).astype(np.uint8)


def decode_np(data, rgb=False):
    """numpy statement of the device decoder: (h, w, 3) uint8 for a YCbCr file, (h, w) for a grayscale one ((h, w, 3) replicated, as
    convert('RGB') gives, with rgb=True).  data: bytes or a path.  Raises ValueError on a file the device does not decode or on
    corrupt entropy-coded data."""
    if isinstance(data, str):
        with open(data, "rb") as f:
            data = f.read()
    h = parse(data)
    if not device_decodable(h):
        raise ValueError("not a file the device decodes (progressive, arithmetic, 12-bit, CMYK, RGB-coded, multi-scan or other sampling)")
    quant = h.scan_tables[0]
    coefs = _huffman_np(h, data)
    planes = []
    hm, vm = _sampling(h)
    for c, (g, blocks) in enumerate(zip(_component_geometry(h), coefs)):
        hs, vs, bw, bh, cw, ch = g
        px = idct_islow_np(blocks.reshape(-1, 64), quant[h.components[c][3]])
        plane = px.reshape(bh, bw, 8, 8).transpose(0, 2, 1, 3).reshape(bh * 8, bw * 8)
        planes.append(upsample_np(plane, cw, ch, hm // hs, vm // vs, h.width, h.height))
    if len(planes) == 1:
        return np.repeat(planes[0][..., None], 3, -1) if rgb else np.ascontiguousarray(planes[0])
    return ycc_to_rgb_np(*planes)


# ------------------------------------------------------------------------------------------------ device

class Image(ctypes.Structure):
    """include/hrviton_sm100_jpeg.h's hrv_jpeg_image."""
    _fields_ = [("data", ctypes.c_int64), ("coef", ctypes.c_int64), ("plane", ctypes.c_int64), ("dst", ctypes.c_uint64),
                ("seg0", ctypes.c_int32), ("nseg", ctypes.c_int32), ("height", ctypes.c_int32), ("width", ctypes.c_int32),
                ("ncomp", ctypes.c_int32), ("hmax", ctypes.c_int32), ("vmax", ctypes.c_int32), ("mcus_x", ctypes.c_int32),
                ("mcus_y", ctypes.c_int32), ("restart", ctypes.c_int32), ("out_channels", ctypes.c_int32),
                ("bw", ctypes.c_int32 * 3), ("bh", ctypes.c_int32 * 3), ("quant", (ctypes.c_uint16 * 64) * 3),
                ("bits", (ctypes.c_uint8 * 16) * 6), ("vals", (ctypes.c_uint8 * 256) * 6)]


class Compact:
    """What the device needs of one file, without the file: the descriptor fields, tables, and its entropy-coded bytes with the
    segment offsets relative to them.  Small and picklable: the loader's workers ship it instead of decoded pixels."""

    def __init__(self, h, data, name="image"):
        self.name = name  # named in the error a corrupt file raises
        s0, s1 = h.segment
        self.entropy = np.frombuffer(data, np.uint8)[s0:s1].copy()
        self.nbytes = s1 - s0
        self.segs = np.array([(a - s0, b - a) for a, b in entropy_segments(h)], np.int32)
        self.height, self.width, self.ncomp = h.height, h.width, len(h.components)
        self.hmax, self.vmax = _sampling(h)
        self.mcus = _mcus(h)
        quant, huff, ri = h.scan_tables
        self.restart = ri
        self.geometry = _component_geometry(h)
        _, td, ta = h.scans[0][:3]
        self.quant = np.stack([quant[c[3]] for c in h.components])
        self.tables = [huff[(0, td[c])] for c in range(self.ncomp)], [huff[(1, ta[c])] for c in range(self.ncomp)]

    @property
    def shape(self):
        return (self.height, self.width) if self.ncomp == 1 else (self.height, self.width, 3)

    def coef_count(self):
        return sum(g[2] * g[3] for g in self.geometry) * 64

    def plane_bytes(self):
        return sum(_align(g[2] * g[3] * 64) for g in self.geometry)


def _align(n, a=16):
    return (n + a - 1) // a * a


def compact(data, name="image"):
    """Compact of a device-decodable file (bytes), or None when the file stays on PIL."""
    h = parse(data)
    return Compact(h, data, name) if device_decodable(h) else None


DESCRIPTOR_BYTES = ctypes.sizeof(Image)


def pack_entropy(items):
    """The entropy-coded bytes of `items` (Compacts) in one uint8 tensor, each image's bytes 16-byte aligned at the offset Batch gives
    it.  The items keep their byte count only."""
    total = sum(_align(c.nbytes) for c in items)
    out = torch.zeros(max(total, 1), dtype=torch.uint8)
    o = 0
    for c in items:
        if c.entropy is not None:
            out[o:o + c.nbytes] = torch.from_numpy(c.entropy)
            c.entropy = None
        o += _align(c.nbytes)
    return out


class Batch:
    """A batch of Compacts packed for one launch of each stage: the descriptor array, segment table and entropy bytes (data: what
    pack_entropy made of the same items, or None to pack them here), plus the sizes of the device scratch (coefficients, planes)."""

    def __init__(self, items, data=None):
        self.items = list(items)
        n = len(self.items)
        self.images = (Image * n)()
        data_off, coef_off, plane_off, seg0 = 0, 0, 0, 0
        segs = []
        self.max_blocks = self.max_pixels = 1
        for i, c in enumerate(self.items):
            d = self.images[i]
            d.data, d.coef, d.plane, d.seg0, d.nseg = data_off, coef_off, plane_off, seg0, len(c.segs)
            d.height, d.width, d.ncomp, d.hmax, d.vmax = c.height, c.width, c.ncomp, c.hmax, c.vmax
            d.mcus_x, d.mcus_y, d.restart, d.out_channels = c.mcus[0], c.mcus[1], c.restart, 1 if c.ncomp == 1 else 3
            for k, g in enumerate(c.geometry):
                d.bw[k], d.bh[k] = g[2], g[3]
                self.max_blocks = max(self.max_blocks, g[2] * g[3])
                ctypes.memmove(d.quant[k], c.quant[k].astype(np.uint16).ctypes.data, 128)
                for slot, (bits, vals) in ((2 * k, c.tables[0][k]), (2 * k + 1, c.tables[1][k])):
                    ctypes.memmove(d.bits[slot], bits.astype(np.uint8).ctypes.data, 16)
                    ctypes.memmove(d.vals[slot], vals.astype(np.uint8).ctypes.data, len(vals))
            self.max_pixels = max(self.max_pixels, c.height * c.width)
            segs.append(c.segs)
            data_off += _align(c.nbytes)
            coef_off += c.coef_count()
            plane_off += c.plane_bytes()
            seg0 += len(c.segs)
        self.data_bytes, self.coef_count, self.plane_bytes = data_off, coef_off, plane_off
        self.segs = torch.from_numpy(np.concatenate(segs).reshape(-1)) if segs else torch.zeros(0, dtype=torch.int32)
        self.data = pack_entropy(self.items) if data is None else data

    def set_destinations(self, dsts):
        """dsts: one contiguous uint8 CUDA tensor per image, of the image's shape, or (h, w, 3) for a grayscale image that is to be
        replicated to RGB."""
        for d, c, t in zip(self.images, self.items, dsts):
            want3 = (c.height, c.width, 3)
            if not (t.is_cuda and t.dtype == torch.uint8 and t.is_contiguous() and tuple(t.shape) in (c.shape, want3)):
                raise ValueError("jpeg: destination %s %s for a %s image" % (t.dtype, tuple(t.shape), c.shape))
            d.dst, d.out_channels = t.data_ptr(), 3 if t.dim() == 3 else 1

    def launch(self, device, stream=None, events=None):
        """Uploads the batch and enqueues the three stages on `stream` (default: the current stream).  Returns the int32 per-image
        error codes on the device (0: decoded).  events: four CUDA events recorded around the stages (timing)."""
        n = len(self.items)
        stream = torch.cuda.current_stream(device) if stream is None else stream
        L, st = capi.lib(), stream.cuda_stream
        with torch.cuda.stream(stream):
            desc = torch.frombuffer(bytearray(bytes(self.images)), dtype=torch.uint8).pin_memory().to(device, non_blocking=True)
            data = (self.data if self.data.is_pinned() else self.data.pin_memory()).to(device, non_blocking=True)
            segs = self.segs.pin_memory().to(device, non_blocking=True)
            coefs = torch.empty(max(self.coef_count, 1), dtype=torch.int16, device=device)
            planes = torch.empty(max(self.plane_bytes, 1), dtype=torch.uint8, device=device)
            errors = torch.zeros(n, dtype=torch.int32, device=device)
            ev = events or [None] * 4
            if ev[0] is not None:
                ev[0].record(stream)
            capi.check(L.hrv_jpeg_huffman(desc.data_ptr(), n, data.data_ptr(), segs.data_ptr(), coefs.data_ptr(), errors.data_ptr(), st),
                       "jpeg_huffman")
            if ev[1] is not None:
                ev[1].record(stream)
            capi.check(L.hrv_jpeg_idct(desc.data_ptr(), n, coefs.data_ptr(), planes.data_ptr(), self.max_blocks, st), "jpeg_idct")
            if ev[2] is not None:
                ev[2].record(stream)
            capi.check(L.hrv_jpeg_color(desc.data_ptr(), n, planes.data_ptr(), self.max_pixels, st), "jpeg_color")
            if ev[3] is not None:
                ev[3].record(stream)
        return errors


def raise_errors(errors, names):
    """Raises OSError naming the first image whose code in `errors` (host int32 array) is not 0."""
    bad = np.flatnonzero(np.asarray(errors))
    if len(bad):
        i = int(bad[0])
        raise OSError("%s: %s" % (names[i], _ERRORS.get(int(errors[i]), "decode error %d" % int(errors[i]))))


def decode(sources, device=None, rgb=False, out=None):
    """Decodes JPEG files on the GPU, bit-identical to PIL's np.asarray(Image.open(f)): a list of uint8 CUDA tensors, (h, w, 3) for a
    YCbCr file and (h, w) for a grayscale one ((h, w, 3), as convert('RGB') gives, with rgb=True).  sources: paths or bytes (or one
    of them).  out: a destination tensor per image to write into instead (the result then is `out`).  Every file must be
    device_decodable (ValueError otherwise); corrupt entropy-coded data raises OSError naming the file.  Synchronises."""
    single = isinstance(sources, (str, bytes, bytearray))
    sources = [sources] if single else list(sources)
    device = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
    items, names = [], []
    for k, s in enumerate(sources):
        name = s if isinstance(s, str) else "image %d" % k
        if isinstance(s, str):
            with open(s, "rb") as f:
                s = f.read()
        c = compact(bytes(s), name)
        if c is None:
            raise ValueError("%s: not a file the device decodes; decode it with PIL" % name)
        items.append(c)
        names.append(name)
    if out is None:
        out = [torch.empty(c.shape if not (rgb and c.ncomp == 1) else (c.height, c.width, 3), dtype=torch.uint8, device=device)
               for c in items]
    b = Batch(items)
    b.set_destinations(out)
    errors = b.launch(device).cpu().numpy()
    raise_errors(errors, names)
    return out[0] if single else out
