"""PNG oracle for the decoder tests: a decoder built on the standard library's zlib plus numpy, and an encoder that can force a filter
type per row, pick the zlib level and strategy, split the stream into IDAT chunks of any size and insert ancillary chunks.  Needs neither
cv2 nor PIL.  Decoding follows cv::imread: IMREAD_COLOR gives BGR (grey replicated, alpha stripped, high byte of 16-bit samples),
IMREAD_GRAYSCALE of a grey or grey + alpha file gives the grey sample."""
from __future__ import annotations

import struct
import zlib

import numpy as np

SIG = b"\x89PNG\r\n\x1a\n"
CHANNELS = {0: 1, 2: 3, 4: 2, 6: 4}


def chunk(kind: bytes, data: bytes) -> bytes:
    return struct.pack(">I", len(data)) + kind + data + struct.pack(">I", zlib.crc32(kind + data) & 0xFFFFFFFF)


def _paeth(a, b, c):
    p = a + b - c
    pa, pb, pc = np.abs(p - a), np.abs(p - b), np.abs(p - c)
    return np.where((pa <= pb) & (pa <= pc), a, np.where(pb <= pc, b, c))


def filter_rows(raw: np.ndarray, bpp: int, filters) -> bytes:
    """raw: rows x rowbytes uint8; filters: one type (0-4) per row."""
    raw = raw.astype(np.int32)
    rows, rb = raw.shape
    out = bytearray()
    for r in range(rows):
        cur = raw[r]
        up = raw[r - 1] if r else np.zeros(rb, np.int32)
        left = np.concatenate([np.zeros(bpp, np.int32), cur[:-bpp]]) if rb > bpp else np.zeros(rb, np.int32)
        ul = np.concatenate([np.zeros(bpp, np.int32), up[:-bpp]]) if rb > bpp else np.zeros(rb, np.int32)
        if rb <= bpp:
            left = np.zeros(rb, np.int32)
            ul = np.zeros(rb, np.int32)
        ft = int(filters[r])
        pred = [np.zeros(rb, np.int32), left, up, (left + up) >> 1, _paeth(left, up, ul)][ft]
        out.append(ft)
        out += ((cur - pred) & 255).astype(np.uint8).tobytes()
    return bytes(out)


def encode(img: np.ndarray, color_type: int, bit_depth: int = 8, filters=None, level: int = 6, strategy: int = zlib.Z_DEFAULT_STRATEGY,
           idat_size: int | None = None, ancillary=(), seed: int = 0) -> bytes:
    """img: rows x cols [x channels] of uint8 or uint16 samples (in file order: grey, RGB, grey + alpha, RGBA).  filters: None (random per
    row from seed), an int (every row), or a sequence.  idat_size: split the zlib stream into IDAT chunks of that many bytes.  ancillary:
    (type, data) chunks inserted between IHDR and the first IDAT."""
    ch = CHANNELS[color_type]
    a = np.asarray(img)
    rows, cols = a.shape[:2]
    a = a.reshape(rows, cols, ch)
    if bit_depth == 16:
        raw = a.astype(">u2").view(np.uint8).reshape(rows, cols * ch * 2)
    else:
        raw = a.astype(np.uint8).reshape(rows, cols * ch)
    bpp = ch * bit_depth // 8
    if filters is None:
        filters = np.random.default_rng(seed).integers(0, 5, rows)
    elif np.isscalar(filters):
        filters = [int(filters)] * rows
    co = zlib.compressobj(level, zlib.DEFLATED, 15, 9, strategy)
    z = co.compress(filter_rows(raw, bpp, filters)) + co.flush()
    out = SIG + chunk(b"IHDR", struct.pack(">IIBBBBB", cols, rows, bit_depth, color_type, 0, 0, 0))
    for kind, data in ancillary:
        out += chunk(kind, data)
    step = idat_size or len(z)
    for i in range(0, len(z), step):
        out += chunk(b"IDAT", z[i : i + step])
    return out + chunk(b"IEND", b"")


def chunks(png: bytes):
    pos, out = 8, []
    while pos + 12 <= len(png):
        (n,) = struct.unpack(">I", png[pos : pos + 4])
        out.append((png[pos + 4 : pos + 8], png[pos + 8 : pos + 8 + n]))
        pos += 12 + n
    return out


def info(png: bytes):
    ihdr = chunks(png)[0][1]
    cols, rows, bd, ct = struct.unpack(">IIBB", ihdr[:10])
    return rows, cols, ct, bd


def zstream(png: bytes) -> bytes:
    return b"".join(d for k, d in chunks(png) if k == b"IDAT")


def with_zstream(png: bytes, z: bytes) -> bytes:
    """the same file with its image data replaced by z (one IDAT chunk)"""
    out = SIG
    done = False
    for k, d in chunks(png):
        if k == b"IDAT":
            if not done:
                out += chunk(b"IDAT", z)
                done = True
            continue
        out += chunk(k, d)
    return out


def unfilter(png: bytes) -> np.ndarray:
    """rows x rowbytes unfiltered samples (bytes as stored, 16-bit big-endian)"""
    rows, cols, ct, bd = info(png)
    bpp = CHANNELS[ct] * bd // 8
    rb = cols * bpp
    data = np.frombuffer(zlib.decompress(zstream(png)), np.uint8).reshape(rows, rb + 1)
    out = np.zeros((rows, rb), np.int32)
    for r in range(rows):
        ft, cur = int(data[r, 0]), data[r, 1:].astype(np.int32)
        up = out[r - 1] if r else np.zeros(rb, np.int32)
        if ft in (0, 2):
            out[r] = (cur + (up if ft == 2 else 0)) & 255
            continue
        row = np.zeros(rb, np.int32)
        for x in range(rb):
            a = row[x - bpp] if x >= bpp else 0
            c = up[x - bpp] if x >= bpp else 0
            b = up[x]
            if ft == 1:
                p = a
            elif ft == 3:
                p = (a + b) >> 1
            else:
                pp = a + b - c
                pa, pb, pc = abs(pp - a), abs(pp - b), abs(pp - c)
                p = a if (pa <= pb and pa <= pc) else (b if pb <= pc else c)
            row[x] = (cur[x] + p) & 255
        out[r] = row
    return out.astype(np.uint8)


def imread(png: bytes, channels: int = 3) -> np.ndarray:
    """cv2.imread(path, IMREAD_COLOR) for channels = 3, IMREAD_GRAYSCALE (grey / grey + alpha files) for channels = 1"""
    rows, cols, ct, bd = info(png)
    s = unfilter(png).reshape(rows, cols, CHANNELS[ct], bd // 8)[..., 0]  # high byte of every sample
    return convert(s, ct, 8, channels)


def convert(samples: np.ndarray, color_type: int, bit_depth: int, channels: int = 3) -> np.ndarray:
    """imread's conversion of rows x cols [x channels] samples as given to encode()"""
    ch = CHANNELS[color_type]
    s = np.asarray(samples)
    s = s.reshape(s.shape[0], s.shape[1], ch)
    s = (s >> 8).astype(np.uint8) if bit_depth == 16 else s.astype(np.uint8)
    if channels == 1:
        assert ch <= 2, "1-channel output is only defined for grey and grey + alpha files"
        return np.ascontiguousarray(s[..., 0])
    if ch <= 2:
        return np.ascontiguousarray(np.repeat(s[..., :1], 3, axis=2))
    return np.ascontiguousarray(s[..., 2::-1])
