"""8-bit RGB PNG encoding on the GPU, pixel-exact, and the multi-task grid of the reference's test_condition.py.

encode() writes a PNG file per image of a CUDA uint8 (N, H, W, 3) batch through the kernels of include/hrviton_sm100_png.h; encode_np()
is the same encoder in numpy, the CPU oracle of the device bytes.  The files decode to the input exactly; their bytes are this
encoder's own (zlib's lazy LZ77 matcher, which PIL runs, is serial and is not reproduced).  The encoder:

    filtering   Paeth (type 4) on every scanline
    chunks      the filtered stream is cut into CHUNK_BYTES-byte pieces (the last one shorter); each is compressed on its own
    matching    RLE only, greedy: each maximal run of equal bytes inside a chunk is one literal, then matches of distance 1 and
                length min(258, rest) while at least 3 bytes are left, then the 1 or 2 bytes left as literals (zlib's Z_RLE)
    coding      one dynamic Huffman block per chunk, code lengths limited to 15 bits (7 for the code-length code) by halving the
                frequencies until the Huffman code fits; a stored block instead when that is not smaller
    joining     a chunk that is not the last ends its Huffman block with an empty stored block (the sync flush: byte alignment);
                only the last chunk's last block sets BFINAL
    framing     one IDAT per chunk, the zlib header (78 01) at the start of the first, the Adler-32 of the filtered stream at the
                end of the last; IHDR and IEND are written on the host

condition_grid() makes test_condition.py's 12-panel grid (make_grid(nrow=4) + save_image's uint8 conversion) on the device;
condition_grid_np() states it in numpy."""
import ctypes
import struct
import zlib

import numpy as np
import torch

from . import capi

SIGNATURE = b"\x89PNG\r\n\x1a\n"
CHUNK_BYTES = 65535              # filtered bytes per chunk: what one stored block holds
ZLIB_HEADER = b"\x78\x01"        # deflate, 32K window, FLEVEL 0 (CMF * 256 + FLG divisible by 31)
MAX_BITS, MAX_CL_BITS = 15, 7
CL_ORDER = (16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15)
LEN_BASE = np.array([3, 4, 5, 6, 7, 8, 9, 10, 11, 13, 15, 17, 19, 23, 27, 31, 35, 43, 51, 59, 67, 83, 99, 115, 131, 163, 195, 227, 258])
LEN_EXTRA = np.array([0, 0, 0, 0, 0, 0, 0, 0, 1, 1, 1, 1, 2, 2, 2, 2, 3, 3, 3, 3, 4, 4, 4, 4, 5, 5, 5, 5, 0])
LEN_SYM = np.searchsorted(LEN_BASE, np.arange(259), side="right") - 1  # length -> index into LEN_BASE (lengths 3..258)
CL_EXTRA = {16: 2, 17: 3, 18: 7}
ADLER_MOD = 65521


# ------------------------------------------------------------------------------------------------ host pieces

def _chunk(kind, payload):
    return struct.pack(">I", len(payload)) + kind + payload + struct.pack(">I", zlib.crc32(kind + payload))


def header(height, width):
    """The signature and IHDR: 8-bit RGB (colour type 2), deflate, adaptive filtering, no interlace."""
    return SIGNATURE + _chunk(b"IHDR", struct.pack(">IIBBBBB", width, height, 8, 2, 0, 0, 0))


TRAILER = _chunk(b"IEND", b"")


def check_encodable(images):
    """(n, h, w) of an encode() / encode_np() batch: uint8 (N, H, W, 3), N, H, W >= 1.  ValueError otherwise."""
    shape, dtype = tuple(images.shape), str(images.dtype).replace("torch.", "")
    if dtype != "uint8" or len(shape) != 4 or shape[3] != 3 or min(shape[:3]) < 1:
        raise ValueError("png.encode: need a uint8 (N, H, W, 3) RGB batch with N, H, W >= 1, got %s %s" % (dtype, shape))
    if shape[1] > 0x7FFFFFFF or shape[2] * 3 + 1 > 0x7FFFFFFF:
        raise ValueError("png.encode: image too large, got %dx%d" % (shape[2], shape[1]))
    return shape[:3]


# ------------------------------------------------------------------------------------------------ numpy oracle

def paeth_np(rgb):
    """The filtered stream of one (H, W, 3) uint8 image: each scanline as the filter type byte 4 and its Paeth residuals."""
    x = rgb.reshape(rgb.shape[0], -1).astype(np.int16)
    a = np.zeros_like(x)
    a[:, 3:] = x[:, :-3]
    b = np.zeros_like(x)
    b[1:] = x[:-1]
    c = np.zeros_like(x)
    c[1:, 3:] = x[:-1, :-3]
    p = a + b - c
    pa, pb, pc = np.abs(p - a), np.abs(p - b), np.abs(p - c)
    pred = np.where((pa <= pb) & (pa <= pc), a, np.where(pb <= pc, b, c))
    out = np.empty((x.shape[0], x.shape[1] + 1), np.uint8)
    out[:, 0] = 4
    out[:, 1:] = (x - pred).astype(np.uint8)
    return out.reshape(-1)


def tokens_np(f):
    """The RLE tokens of one chunk f (uint8): (position, length) of each, length 0 for a literal (the byte at position) and 3..258
    for a match of distance 1 starting at position."""
    n = len(f)
    start = np.ones(n, bool)
    start[1:] = f[1:] != f[:-1]
    starts = np.flatnonzero(start)
    run = np.cumsum(start) - 1
    s = starts[run]
    e = np.append(starts[1:], n)[run]
    k = np.arange(n) - s
    r = e - s
    km = np.maximum(k, 1)
    base = km - (km - 1) % 258
    mlen = np.minimum(258, r - base)
    literal = (k == 0) | (mlen < 3)
    match = (k > 0) & (mlen >= 3) & (k == base)
    pos = np.flatnonzero(literal | match)
    return pos, np.where(match[pos], mlen[pos], 0)


def huffman_lengths(freq, limit):
    """Code lengths of a Huffman code for freq (symbols with freq 0 get no code), at most `limit` bits.  Deterministic: leaves in
    (freq, symbol) order, the two-queue merge taking a leaf when its frequency is <= the internal node's; when the code is too long,
    every nonzero frequency f becomes (f + 1) >> 1 and the code is built again.  One used symbol: it and the lowest other symbol get
    length 1 (inflate takes only complete code-length codes)."""
    f = [int(v) for v in freq]
    lengths = [0] * len(f)
    used = [s for s in range(len(f)) if f[s] > 0]
    if len(used) == 1:
        lengths[used[0]] = 1
        lengths[1 if used[0] == 0 else 0] = 1
        return lengths
    while True:
        leaves = sorted(used, key=lambda s: (f[s], s))
        m = len(leaves)
        parent = [0] * (2 * m - 1)
        nf = [f[s] for s in leaves] + [0] * (m - 1)
        i, j = 0, m
        for t in range(m, 2 * m - 1):
            pair = []
            for _ in range(2):
                if i < m and (j >= t or nf[i] <= nf[j]):
                    pair.append(i)
                    i += 1
                else:
                    pair.append(j)
                    j += 1
            nf[t] = nf[pair[0]] + nf[pair[1]]
            parent[pair[0]] = parent[pair[1]] = t
        depth = [0] * (2 * m - 1)
        for t in range(2 * m - 3, -1, -1):
            depth[t] = depth[parent[t]] + 1
        if max(depth[:m]) <= limit:
            for q, s in enumerate(leaves):
                lengths[s] = depth[q]
            return lengths
        f = [(v + 1) >> 1 if v else 0 for v in f]


def canonical_codes(lengths):
    """RFC 1951 canonical codes of `lengths`, bit-reversed for LSB-first output."""
    lengths = list(lengths)
    mx = max(lengths)
    count = [0] * (mx + 1)
    for n in lengths:
        if n:
            count[n] += 1
    code, nxt = 0, [0] * (mx + 2)
    for b in range(1, mx + 1):
        code = (code + count[b - 1]) << 1 if b > 1 else 0
        nxt[b] = code
    out = [0] * len(lengths)
    for s, n in enumerate(lengths):
        if n:
            c = nxt[n]
            nxt[n] += 1
            out[s] = int("{:0{}b}".format(c, n)[::-1], 2)
    return out


def code_length_items(seq):
    """The code-length alphabet items (symbol, extra) of a sequence of code lengths: runs of zeros as 18 (11..138) then 17 (3..10),
    runs of a nonzero length as the length then 16 (3..6 repeats); what is left of a run as plain lengths."""
    items, i, n = [], 0, len(seq)
    while i < n:
        v, r = seq[i], 1
        while i + r < n and seq[i + r] == v:
            r += 1
        i += r
        if v == 0:
            while r >= 11:
                m = min(r, 138)
                items.append((18, m - 11))
                r -= m
            if r >= 3:
                items.append((17, r - 3))
                r = 0
        else:
            items.append((v, 0))
            r -= 1
            while r >= 3:
                m = min(r, 6)
                items.append((16, m - 3))
                r -= m
        items.extend([(v, 0)] * r)
    return items


def _pack(vals, lens):
    """LSB-first bit packing of (value, length) fields, as bytes padded with zero bits."""
    vals, lens = np.asarray(vals, np.int64), np.asarray(lens, np.int64)
    total = int(lens.sum())
    starts = np.cumsum(lens) - lens
    idx = np.repeat(np.arange(len(lens)), lens)
    j = np.arange(total) - starts[idx]
    bits = ((vals[idx] >> j) & 1).astype(np.uint8)
    return np.packbits(bits, bitorder="little").tobytes(), total


def deflate_chunk_np(f, final):
    """The deflate bytes of one chunk (byte-aligned at both ends): a dynamic Huffman block of its RLE tokens, then, unless final, an
    empty stored block; or one stored block when that is not larger."""
    f = np.asarray(f, np.uint8)
    n = len(f)
    stored = bytes([1 if final else 0]) + struct.pack("<HH", n, n ^ 0xFFFF) + f.tobytes()
    pos, mlen = tokens_np(f)
    sym = np.where(mlen > 0, 257 + LEN_SYM[mlen], f[pos].astype(np.int64))
    freq = np.bincount(sym, minlength=286)
    freq[256] += 1
    lit_len = huffman_lengths(freq, MAX_BITS)
    nlit = max(257, max(s for s in range(286) if lit_len[s]) + 1)
    items = code_length_items(lit_len[:nlit] + [1])  # one distance code (distance 1) of length 1
    cl_freq = np.bincount([s for s, _ in items], minlength=19)
    cl_len = huffman_lengths(cl_freq, MAX_CL_BITS)
    ncl = max(4, max(q for q in range(19) if cl_len[CL_ORDER[q]]) + 1)
    lit_code, cl_code = canonical_codes(lit_len), canonical_codes(cl_len)
    vals = [1 if final else 0, 2, nlit - 257, 0, ncl - 4] + [cl_len[CL_ORDER[q]] for q in range(ncl)]
    lens = [1, 2, 5, 5, 4] + [3] * ncl
    for s, x in items:
        vals.append(cl_code[s] | (x << cl_len[s]))
        lens.append(cl_len[s] + CL_EXTRA.get(s, 0))
    lit_code, lit_len = np.array(lit_code, np.int64), np.array(lit_len, np.int64)
    li = np.maximum(sym - 257, 0)
    ext = np.where(mlen > 0, LEN_EXTRA[li], 0)
    xv = np.where(mlen > 0, mlen - LEN_BASE[li], 0)
    # code, extra bits, then the distance code (a single 0 bit) for a match
    tv = lit_code[sym] | (xv << lit_len[sym])
    tl = lit_len[sym] + ext + (mlen > 0)
    vals = np.concatenate([vals, tv, [lit_code[256]]] + ([] if final else [[0]]))
    lens = np.concatenate([lens, tl, [lit_len[256]]] + ([] if final else [[3]]))
    body, _ = _pack(vals, lens)
    dyn = body + (b"" if final else b"\x00\x00\xff\xff")
    return dyn if len(dyn) < len(stored) else stored


def _adler_parts(f):
    f = f.astype(np.int64)
    n = len(f)
    return int(f.sum()) % ADLER_MOD, int(((n - np.arange(n)) * f).sum() % ADLER_MOD)


def encode_one_np(rgb):
    """The PNG file of one (H, W, 3) uint8 image."""
    h, w = rgb.shape[:2]
    stream = paeth_np(np.ascontiguousarray(rgb))
    total = len(stream)
    nchunks = -(-total // CHUNK_BYTES)
    out = [header(h, w)]
    s1, s2 = 1, total % ADLER_MOD
    for c in range(nchunks):
        o = c * CHUNK_BYTES
        f = stream[o:o + CHUNK_BYTES]
        a, b = _adler_parts(f)
        s1 = (s1 + a) % ADLER_MOD
        s2 = (s2 + b + (total - o - len(f)) % ADLER_MOD * a) % ADLER_MOD
        data = (ZLIB_HEADER if c == 0 else b"") + deflate_chunk_np(f, c == nchunks - 1)
        if c == nchunks - 1:
            data += struct.pack(">I", (s2 << 16) | s1)
        out.append(_chunk(b"IDAT", data))
    out.append(TRAILER)
    return b"".join(out)


def encode_np(images):
    """numpy statement of the device encoder: the PNG bytes of every image of a uint8 (N, H, W, 3) RGB batch (or one (H, W, 3)
    image), a list of bytes equal to encode()'s."""
    images = np.asarray(images)
    if images.dtype == np.uint8 and images.ndim == 3:
        images = images[None]
    check_encodable(images)
    return [encode_one_np(rgb) for rgb in images]


# ------------------------------------------------------------------------------------------------ encoding: device

def encode(images, stream=None, stats=None):
    """PNG files of a batch on the GPU: a list of bytes, equal to encode_np's, each decoding to its image exactly.  images: a CUDA
    uint8 (N, H, W, 3) RGB batch, any H, W >= 1 (ValueError otherwise).

    Runs on `stream` (default: the current stream), ordered after the work that wrote `images`.  The device sends back only the IDAT
    chunks: one small copy of the per-image lengths and offsets (the one wait for the device), then one copy of the bytes; the host
    writes the signature, IHDR and IEND.  stats: a dict that receives 'd2h_bytes', the bytes copied from the device."""
    n, h, w = check_encodable(images)
    if not (torch.is_tensor(images) and images.is_cuda):
        raise ValueError("png.encode: need a CUDA tensor (encode_np encodes host arrays)")
    device = images.device
    L = capi.lib()
    ws_bytes, out_bytes = ctypes.c_size_t(), ctypes.c_size_t()
    capi.check(L.hrv_png_encode_bounds(n, h, w, ctypes.byref(ws_bytes), ctypes.byref(out_bytes)), "png_encode_bounds")
    with torch.cuda.device(device):
        stream = torch.cuda.current_stream(device) if stream is None else stream
        with torch.cuda.stream(stream):
            images = images.contiguous()
            ws = torch.empty(ws_bytes.value, dtype=torch.uint8, device=device)
            out = torch.empty(out_bytes.value, dtype=torch.uint8, device=device)
            sizes = torch.empty(2 * n, dtype=torch.int64, device=device)
            capi.check(L.hrv_png_encode(images.data_ptr(), n, h, w, ws.data_ptr(), ws_bytes.value, out.data_ptr(), out_bytes.value,
                                        sizes.data_ptr(), stream.cuda_stream), "png_encode")
            host_sizes = torch.empty(2 * n, dtype=torch.int64, pin_memory=True)
            host_sizes.copy_(sizes, non_blocking=True)
            done = torch.cuda.Event()
            done.record(stream)
            done.synchronize()
            lengths, offsets = host_sizes[0::2].tolist(), host_sizes[1::2].tolist()
            total = offsets[-1] + lengths[-1]
            host = torch.empty(total, dtype=torch.uint8, pin_memory=True)
            host.copy_(out[:total], non_blocking=True)
            done.record(stream)
            done.synchronize()
    if stats is not None:
        stats["d2h_bytes"] = stats.get("d2h_bytes", 0) + total + 16 * n
    head = header(h, w)
    mv = memoryview(host.numpy())
    return [head + mv[o:o + l].tobytes() + TRAILER for o, l in zip(offsets, lengths)]


# ------------------------------------------------------------------------------------------------ the multi-task grid

# utils.visualize_segmap's palette; Image.putpalette leaves the entries past it black
PALETTE = np.zeros((256, 3), np.uint8)
PALETTE[:20] = np.array([0, 0, 0, 128, 0, 0, 254, 0, 0, 0, 85, 0, 169, 0, 51, 254, 85, 0, 0, 0, 85, 0, 119, 220, 85, 85, 0, 0, 85, 85,
                         85, 51, 0, 52, 86, 128, 0, 128, 0, 0, 0, 254, 51, 169, 220, 0, 254, 254, 85, 254, 169, 169, 254, 85, 254, 254, 0,
                         254, 169, 0]).reshape(20, 3)
COMPOSITIONS = {"no_composition": capi.GRID_NO_COMPOSITION, "detach": capi.GRID_DETACH, "warp_grad": capi.GRID_WARP_GRAD}
# the grid's inputs: (name, channels; 0 for the segmentation's class count)
GRID_INPUTS = (("cloth", 3), ("cloth_mask", 1), ("parse_agnostic", 0), ("densepose", 3), ("parse_cloth", 3), ("pcm", 1), ("warped_cloth", 3),
               ("warped_cm", 1), ("parse", 0), ("seg", 0), ("image", 3))


def grid_shape(n, h, w):
    """(N, 3 (H + 2) + 2, 4 (W + 2) + 2, 3): make_grid of 12 panels, nrow 4, padding 2."""
    return n, 3 * (h + 2) + 2, 4 * (w + 2) + 2, 3


def composed_np(seg, warped_cm, composition):
    """test_condition.py:108-117: seg with channel 3 times warped_cm ('warp_grad') or times (warped_cm > 0.5) ('detach'), fp32."""
    seg = np.array(seg, np.float32)
    if composition == "warp_grad":
        seg[:, 3] = seg[:, 3] * warped_cm[:, 0]
    elif composition == "detach":
        seg[:, 3] = seg[:, 3] * (warped_cm[:, 0] > 0.5).astype(np.float32)
    elif composition != "no_composition":
        raise ValueError("composition must be one of %s, got %r" % (sorted(COMPOSITIONS), composition))
    return seg


def condition_grid_np(t, composition="warp_grad"):
    """numpy statement of condition_grid: t maps GRID_INPUTS' names to fp32 NCHW arrays."""
    t = {k: np.asarray(v, np.float32) for k, v in t.items()}
    n, _, h, w = t["cloth"].shape
    f = np.float32
    half = lambda x: x / f(2) + f(0.5)  # noqa: E731
    three = lambda x: np.broadcast_to(x, (n, 3, h, w))  # noqa: E731
    segmap = lambda x: PALETTE[np.argmax(x, axis=1)].transpose(0, 3, 1, 2).astype(np.float32) / f(255)  # noqa: E731
    seg = composed_np(t["seg"], t["warped_cm"], composition)
    wcm1 = (t["warped_cm"] > 0.5).astype(np.float32)
    misalign = np.maximum((np.argmax(seg, axis=1)[:, None] == 3).astype(np.float32) - wcm1, f(0))
    panels = [half(t["cloth"]), three((t["cloth_mask"] > 0.5).astype(np.float32)), segmap(t["parse_agnostic"]), (t["densepose"] + f(1)) / f(2),
              half(t["parse_cloth"]), three(t["pcm"]), half(t["warped_cloth"]), three(wcm1), segmap(t["parse"]), segmap(seg),
              half(t["image"]), three(misalign)]
    grid = np.zeros((n, 3, 3 * (h + 2) + 2, 4 * (w + 2) + 2), np.float32)
    for k, p in enumerate(panels):
        y, x = 2 + (k // 4) * (h + 2), 2 + (k % 4) * (w + 2)
        grid[:, :, y:y + h, x:x + w] = p
    with np.errstate(invalid="ignore"):
        u8 = np.clip(grid * f(255) + f(0.5), 0, 255).astype(np.uint8)
    return u8.transpose(0, 2, 3, 1)


def condition_grid(t, composition="warp_grad", out=None):
    """test_condition.py:135-143's multi-task grid of every sample, on the device, in one launch: uint8 (N, 3 (H + 2) + 2, 4 (W + 2) + 2,
    3), bit for bit what make_grid(12 panels, nrow=4) and save_image's conversion hand to PIL.  t maps GRID_INPUTS' names to CUDA
    fp32 NCHW tensors of one batch and size: cloth, densepose, parse_cloth, warped_cloth, image (3 channels); cloth_mask, pcm,
    warped_cm (1); parse_agnostic, parse and seg (the tocg's segmentation before composition) with one channel per class.  Runs on
    the current stream."""
    missing = [k for k, _ in GRID_INPUTS if k not in t]
    if missing:
        raise KeyError("condition_grid: missing %s" % missing)
    if composition not in COMPOSITIONS:
        raise ValueError("composition must be one of %s, got %r" % (sorted(COMPOSITIONS), composition))
    n, _, h, w = t["cloth"].shape
    classes = t["seg"].shape[1]
    ts = {}
    for k, c in GRID_INPUTS:
        v = t[k]
        want = (n, c or classes, h, w)
        if not (torch.is_tensor(v) and v.is_cuda and v.dtype == torch.float32 and tuple(v.shape) == want):
            raise ValueError("condition_grid: %s must be a CUDA float32 %s tensor, got %s" % (
                k, want, "%s %s %s" % (v.device, v.dtype, tuple(v.shape)) if torch.is_tensor(v) else type(v)))
        ts[k] = v.contiguous()
    if out is None:
        out = torch.empty(grid_shape(n, h, w), dtype=torch.uint8, device=ts["cloth"].device)
    p = capi.ConditionPanels(**{k: v.data_ptr() for k, v in ts.items()})
    capi.check(capi.lib().hrv_condition_grid(ctypes.byref(p), n, h, w, classes, COMPOSITIONS[composition], out.data_ptr(),
                                             torch.cuda.current_stream(out.device).cuda_stream), "condition_grid")
    return out
