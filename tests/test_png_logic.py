"""PNG decoding on the CPU (no GPU): the stdlib oracle against the cv2 goldens, the container walk of the built library
(xivo_png_info), and the decoder code of xivo_b200/csrc/png.cuh compiled with g++ (tests/cpp/png_harness.cpp) against the oracle on a
corpus, on corrupt deflate streams and on random bit flips."""
import ctypes as C
import os
import shutil
import struct
import subprocess
import zlib

import numpy as np
import pytest

import png_oracle as O

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "png_imread.npz")


def goldens():
    g = np.load(GOLDEN)
    for i, name in enumerate(g["names"]):
        yield str(name), g[f"png_{i}"].tobytes(), g[f"color_{i}"], (g[f"gray_{i}"] if f"gray_{i}" in g else None)


def test_oracle_equals_goldens():
    n = 0
    for name, png, color, gray in goldens():
        assert np.array_equal(O.imread(png, 3), color), name
        if gray is not None:
            assert np.array_equal(O.imread(png, 1), gray), name
        n += 1
    assert n >= 16


def test_oracle_equals_live_cv2(tmp_path):
    cv2 = pytest.importorskip("cv2")
    rng = np.random.default_rng(0)
    for ct in (0, 2, 4, 6):
        for bd in (8, 16):
            img = rng.integers(0, 1 << bd, (9, 13, O.CHANNELS[ct]))
            png = O.encode(img, ct, bd, level=rng.integers(0, 10))
            p = str(tmp_path / f"{ct}_{bd}.png")
            open(p, "wb").write(png)
            assert np.array_equal(O.imread(png, 3), cv2.imread(p)), (ct, bd)
            assert np.array_equal(O.convert(img, ct, bd, 3), cv2.imread(p)), (ct, bd)
            if ct in (0, 4):
                assert np.array_equal(O.imread(png, 1), cv2.imread(p, cv2.IMREAD_GRAYSCALE)), (ct, bd)


# ------------------------------------------------------------------------------------------------ xivo_png_info (built library)
@pytest.fixture(scope="module")
def xlib():
    from xivo_b200 import capi

    return capi


def ihdr_png(cols=5, rows=4, bd=8, ct=0, comp=0, filt=0, interlace=0, body=None):
    img = np.zeros((rows, cols, O.CHANNELS.get(ct, 1)), np.uint8)
    good = O.encode(img, 0 if ct not in O.CHANNELS else ct, 8)
    ihdr = struct.pack(">IIBBBBB", cols, rows, bd, ct, comp, filt, interlace)
    return O.SIG + O.chunk(b"IHDR", ihdr) + (body if body is not None else O.chunk(b"IDAT", O.zstream(good)) + O.chunk(b"IEND", b""))


def test_png_info_geometry(xlib):
    for ct in (0, 2, 4, 6):
        for bd in (8, 16):
            png = O.encode(np.zeros((7, 11, O.CHANNELS[ct]), np.uint16), ct, bd)
            assert xlib.png_info(png) == (7, 11, O.CHANNELS[ct], bd)
    for name, png, color, _ in goldens():
        r, c, ch, bd = xlib.png_info(png)
        assert (r, c) == color.shape[:2] and ch == O.CHANNELS[O.info(png)[2]] and bd == O.info(png)[3], name


REFUSALS = [
    ("bad signature", lambda: b"\x89PNX" + ihdr_png()[4:]),
    ("IHDR missing", lambda: O.SIG + O.chunk(b"IDAT", b"x") + O.chunk(b"IEND", b"")),
    ("misplaced IHDR", lambda: ihdr_png(body=O.chunk(b"IHDR", b"\0" * 13) + O.chunk(b"IEND", b""))),
    ("missing IDAT", lambda: ihdr_png(body=O.chunk(b"IEND", b""))),
    ("missing IEND", lambda: ihdr_png(body=O.chunk(b"IDAT", b"x"))),
    ("runs past the end", lambda: ihdr_png(body=struct.pack(">I", 1000) + b"IDAT" + b"xx")),
    ("palette", lambda: ihdr_png(ct=3)),
    ("bit depths below 8", lambda: ihdr_png(bd=4)),
    ("bit depths below 8", lambda: ihdr_png(bd=1)),
    ("bit depths below 8", lambda: ihdr_png(bd=2)),
    ("interlaced", lambda: ihdr_png(interlace=1)),
    ("zero width or height", lambda: ihdr_png(cols=0)),
    ("zero width or height", lambda: ihdr_png(rows=0)),
    ("too large", lambda: ihdr_png(cols=100000)),
    ("invalid colour type", lambda: ihdr_png(ct=5)),
    ("not consecutive", lambda: ihdr_png(body=O.chunk(b"IDAT", b"x") + O.chunk(b"tEXt", b"a\0b") + O.chunk(b"IDAT", b"y") + O.chunk(b"IEND", b""))),
]


@pytest.mark.parametrize("why,make", REFUSALS, ids=[f"{i}_{w.replace(' ', '_')}" for i, (w, _) in enumerate(REFUSALS)])
def test_png_info_refusals(xlib, why, make):
    with pytest.raises(xlib.XivoError, match=why):
        xlib.png_info(make())


def test_png_info_every_truncation_is_refused(xlib):
    png = O.encode(np.arange(60, dtype=np.uint8).reshape(6, 10), 0, 8, ancillary=[(b"gAMA", b"\0\0\xb1\x8f")], idat_size=7)
    assert xlib.png_info(png) == (6, 10, 1, 8)
    for k in range(len(png)):
        with pytest.raises(xlib.XivoError):
            xlib.png_info(png[:k])


# ------------------------------------------------------------------------------------------------ the shared decoder under g++
def _harness(tmp, flags=()):
    so = str(tmp / "libpng_harness.so")
    cmd = ["g++", "-std=c++17", "-O2", *flags, "-shared", "-fPIC", os.path.join(ROOT, "tests", "cpp", "png_harness.cpp"), "-o", so]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    return _load(so)


def _load(so):
    lib = C.CDLL(so)
    lib.ph_info.argtypes = [C.c_char_p, C.c_size_t, C.c_void_p, C.c_char_p, C.c_int]
    lib.ph_inflate.argtypes = [C.c_char_p, C.c_size_t, C.c_void_p, C.c_size_t]
    lib.ph_decode.argtypes = [C.c_char_p, C.c_size_t, C.c_int, C.c_void_p]
    lib.ph_status_text.restype = C.c_char_p
    return lib


@pytest.fixture(scope="module")
def ph(tmp_path_factory):
    so = os.environ.get("XIVO_PNG_HARNESS_SO")  # set by scripts/png_sanitize.sh: the ASan / UBSan build
    if so:
        return _load(so)
    if shutil.which("g++") is None:
        pytest.skip("needs g++")
    return _harness(tmp_path_factory.mktemp("ph"))


def decode(ph, png, oc=3):
    r, c = O.info(png)[:2]
    out = np.zeros((r, c, oc), np.uint8)
    rc = ph.ph_decode(png, len(png), oc, out.ctypes.data)
    return rc, (out if oc == 3 else out[..., 0])


def inflate(ph, z, cap):
    out = np.zeros(max(cap, 1), np.uint8)
    return ph.ph_inflate(z, len(z), out.ctypes.data, cap), out[:cap]


def corpus():
    rng = np.random.default_rng(1)
    items = []
    strategies = [zlib.Z_DEFAULT_STRATEGY, zlib.Z_FILTERED, zlib.Z_HUFFMAN_ONLY, zlib.Z_RLE, zlib.Z_FIXED]
    shapes = [(1, 1), (1, 77), (33, 1), (17, 33), (40, 48)]
    k = 0
    for ct in (0, 2, 4, 6):
        for bd in (8, 16):
            for (r, c) in shapes:
                top = (1 << bd) - 1
                smooth = (np.add.outer(np.arange(r), np.arange(c))[..., None] * (37 + 11 * np.arange(O.CHANNELS[ct]))) % (top + 1)
                img = np.where(rng.random((r, c, O.CHANNELS[ct])) < 0.3, rng.integers(0, top + 1, (r, c, O.CHANNELS[ct])), smooth)
                filt = [None, 0, 1, 2, 3, 4][k % 6]
                png = O.encode(img, ct, bd, filters=filt, level=[0, 1, 6, 9][k % 4], strategy=strategies[k % 5], idat_size=[None, 1, 50][k % 3],
                               seed=k)
                items.append((img, ct, bd, png))
                k += 1
    return items


def test_harness_matches_oracle_on_corpus(ph):
    for img, ct, bd, png in corpus():
        rc, out = decode(ph, png, 3)
        assert rc == 0, ph.ph_status_text(rc)
        assert np.array_equal(out, O.convert(img, ct, bd, 3)), (img.shape, ct, bd)
        if ct in (0, 4):
            rc, out = decode(ph, png, 1)
            assert rc == 0 and np.array_equal(out, O.convert(img, ct, bd, 1))


def test_harness_matches_goldens(ph):
    for name, png, color, gray in goldens():
        rc, out = decode(ph, png, 3)
        assert rc == 0 and np.array_equal(out, color), name
        if gray is not None:
            rc, out = decode(ph, png, 1)
            assert rc == 0 and np.array_equal(out, gray), name


def stored(data, final=1):
    return bytes([final]) + struct.pack("<HH", len(data), 0xFFFF ^ len(data)) + data


def zwrap(deflate, payload):
    return b"\x78\x01" + deflate + struct.pack(">I", zlib.adler32(payload))


def _bits(fields):
    """deflate bit string from (value, nbits) fields, LSB first"""
    acc, n, out = 0, 0, bytearray()
    for v, k in fields:
        acc |= v << n
        n += k
    while n > 0:
        out.append(acc & 255)
        acc >>= 8
        n -= 8
    return bytes(out)


def _dyn_header(hlit, hdist, hclen, cl_lens):
    f = [(1, 1), (2, 2), (hlit - 257, 5), (hdist - 1, 5), (hclen - 4, 4)]
    return f + [(v, 3) for v in cl_lens[:hclen]]


def _corrupt_cases():
    payload = bytes(range(200)) * 3
    good = zlib.compress(payload, 6)
    cases = {
        "truncated": (good[: len(good) // 2], len(payload), "truncated"),
        "block_type_3": (b"\x78\x01" + bytes([0b111]) + b"\0" * 8, 10, "block type 3"),
        "stored_len_nlen": (b"\x78\x01" + bytes([1]) + struct.pack("<HH", 5, 5) + b"abcde" + b"\0" * 4, 5, "complement"),
        # dynamic header: code-length code lengths all 1 for 19 symbols -> over-subscribed
        "oversubscribed": (b"\x78\x01" + _bits(_dyn_header(257, 1, 19, [1] * 19)) + b"\0" * 8, 10, "over-subscribed"),
        # a single code-length code of length 2 -> incomplete
        "incomplete": (b"\x78\x01" + _bits(_dyn_header(257, 1, 4, [2, 0, 0, 0])) + b"\0" * 8, 10, "incomplete"),
        "hlit_gt_286": (b"\x78\x01" + _bits(_dyn_header(287, 1, 4, [1, 1, 0, 0])) + b"\0" * 8, 10, "HLIT"),
        "hdist_gt_30": (b"\x78\x01" + _bits(_dyn_header(257, 31, 4, [1, 1, 0, 0])) + b"\0" * 8, 10, "HDIST"),
        # fixed block: literal 'a' then a match of length 3 at distance 2 (only 1 byte written)
        "distance_too_far": (b"\x78\x01" + _fixed([("lit", 97), ("match", 3, 2), ("eob",)]) + b"\0" * 4, 10, "too far back"),
        "bad_adler": (good[:-4] + struct.pack(">I", (zlib.adler32(payload) ^ 1)), len(payload), "Adler"),
        "too_few_bytes": (good, len(payload) + 1, "too little"),
        "too_many_bytes": (good, len(payload) - 1, "too much"),
        "bad_zlib_header": (b"\x79\x01" + good[2:], len(payload), "zlib header"),
        "preset_dictionary": (bytes([0x78, 0x20 | (31 - ((0x78 << 8 | 0x20) % 31))]) + good[2:], len(payload), "zlib header"),
    }
    return cases


def _fixed(tokens):
    """fixed-Huffman block from tokens (final block)"""
    f = [(1, 1), (1, 2)]

    def rev(v, n):
        return int(format(v, f"0{n}b")[::-1], 2)

    def lit(sym):
        if sym < 144:
            return rev(0x30 + sym, 8), 8
        if sym < 256:
            return rev(0x190 + sym - 144, 9), 9
        if sym < 280:
            return rev(sym - 256, 7), 7
        return rev(0xC0 + sym - 280, 8), 8

    for t in tokens:
        if t[0] == "lit":
            f.append(lit(t[1]))
        elif t[0] == "eob":
            f.append(lit(256))
        else:
            _, length, dist = t
            assert 3 <= length <= 10 and 1 <= dist <= 4
            f.append(lit(257 + length - 3))
            f.append((rev(dist - 1, 5), 5))
    return _bits(f)


@pytest.mark.parametrize("name", sorted(_corrupt_cases()))
def test_harness_rejects_corrupt_streams(ph, name):
    z, cap, why = _corrupt_cases()[name]
    rc, _ = inflate(ph, z, cap)
    assert rc != 0
    assert why.lower() in ph.ph_status_text(rc).decode().lower(), (name, ph.ph_status_text(rc))


def test_harness_fixed_and_stored_blocks_decode(ph):
    z = b"\x78\x01" + _fixed([("lit", 97), ("lit", 98), ("match", 6, 2), ("eob",)])
    z += struct.pack(">I", zlib.adler32(b"abababab"))
    rc, out = inflate(ph, z, 8)
    assert rc == 0 and out.tobytes() == b"abababab"
    payload = b"hello stored"
    rc, out = inflate(ph, zwrap(stored(payload), payload), len(payload))
    assert rc == 0 and out.tobytes() == payload
    rc, _ = inflate(ph, zwrap(stored(payload)[:-1], payload), len(payload))
    assert rc != 0


def test_harness_every_truncation_fails(ph):
    payload = np.random.default_rng(3).integers(0, 4, 3000).astype(np.uint8).tobytes()
    for level in (0, 1, 9):
        z = zlib.compress(payload, level)
        for k in range(len(z)):
            rc, _ = inflate(ph, z[:k], len(payload))
            assert rc != 0, (level, k)


def test_harness_random_bit_flips_stay_in_bounds(ph):
    """flipped bits may decode or fail; the harness writes only inside its buffers (checked under ASan by scripts/png_sanitize.sh)"""
    rng = np.random.default_rng(4)
    payload = rng.integers(0, 8, 5000).astype(np.uint8).tobytes()
    z = bytearray(zlib.compress(payload, 6))
    fails = 0
    for i in range(600):
        b = bytearray(z)
        for _ in range(1 + i % 3):
            pos = int(rng.integers(0, len(b)))
            b[pos] ^= 1 << int(rng.integers(0, 8))
        cap = len(payload) + int(rng.integers(-3, 4))
        rc, _ = inflate(ph, bytes(b), cap)
        fails += rc != 0
    assert fails > 500


def test_harness_under_sanitizers(tmp_path):
    """the harness compiled with -fsanitize=address,undefined runs the corpus, the corrupt set and bit flips in a child process"""
    if shutil.which("g++") is None:
        pytest.skip("needs g++")
    script = os.path.join(ROOT, "scripts", "png_sanitize.sh")
    r = subprocess.run(["bash", script], capture_output=True, text=True, cwd=ROOT, env=dict(os.environ, PNG_SAN_DIR=str(tmp_path)))
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    assert "sanitizers: no report" in r.stdout
