"""PNG decoding on the device (png_inflate_kernel, png_unfilter_kernel) against the stdlib oracle and the cv2 goldens, and PNG ingest
through pyxivo: Batch.visual_meas_png and Estimator.VisualMeas(ts, path) must give bit-identical results to feeding the decoded arrays,
and refused frames must leave every sequence untouched."""
import os
import zlib

import numpy as np
import pytest

import png_oracle as O
from xivo_b200 import XivoError, pyxivo, sim

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CFG = os.path.join(ROOT, "xivo_b200", "cfg")
GOLDEN = os.path.join(ROOT, "tests", "golden", "png_imread.npz")
STRATEGIES = [zlib.Z_DEFAULT_STRATEGY, zlib.Z_FILTERED, zlib.Z_HUFFMAN_ONLY, zlib.Z_RLE, zlib.Z_FIXED]


def textured(rng, rows, cols, ch, bits):
    top = (1 << bits) - 1
    y, x = np.mgrid[0:rows, 0:cols]
    base = (np.sin(x / 7.0 + rng.random() * 6) * np.cos(y / 5.0) * 0.45 + 0.5)[..., None] * top * (0.5 + 0.5 * np.arange(1, ch + 1) / ch)
    noise = rng.integers(0, max(top // 16, 2), (rows, cols, ch))
    img = np.clip(base + noise, 0, top)
    return img.astype(np.uint16 if bits == 16 else np.uint8)


def mixed_corpus(n_small=260):
    """(samples, colour type, bit depth, png) of mixed geometry, levels, strategies, filters and IDAT splits"""
    rng = np.random.default_rng(7)
    out = []
    big = [((480, 752), 0, 8), ((512, 512), 0, 16), ((480, 640), 2, 8), ((240, 320), 6, 16)]
    for k, ((r, c), ct, bd) in enumerate(big * 2):
        img = textured(rng, r, c, O.CHANNELS[ct], bd)
        out.append((img, ct, bd, O.encode(img, ct, bd, filters=[None, 4, 1, 3][k % 4], level=[1, 6, 9, 0][k % 4], strategy=STRATEGIES[k % 5],
                                          idat_size=[None, 8192][k % 2], seed=k)))
    shapes = [(1, 1), (1, 777), (333, 1), (17, 33), (31, 64), (8, 8)]
    for k in range(n_small):
        r, c = shapes[k % len(shapes)]
        ct, bd = [(0, 8), (0, 16), (2, 8), (2, 16), (4, 8), (4, 16), (6, 8), (6, 16)][(k // len(shapes)) % 8]
        img = textured(rng, r, c, O.CHANNELS[ct], bd)
        filt = [None, 0, 1, 2, 3, 4][k % 6]
        png = O.encode(img, ct, bd, filters=filt, level=[0, 1, 6, 9][k % 4], strategy=STRATEGIES[(k // 4) % 5], idat_size=[None, 1, 8192][k % 3],
                       seed=k)
        out.append((img, ct, bd, png))
    return out


def test_decode_png_matches_oracle_mixed_geometry(ctx):
    corpus = mixed_corpus()
    assert len(corpus) >= 256
    got = ctx.decode_png([p for *_, p in corpus], 3)
    for i, ((img, ct, bd, _), g) in enumerate(zip(corpus, got)):
        assert np.array_equal(g, O.convert(img, ct, bd, 3)), (i, img.shape, ct, bd)
    grey = [(img, ct, bd, p) for img, ct, bd, p in corpus if ct in (0, 4)]
    got = ctx.decode_png([p for *_, p in grey], 1)
    for (img, ct, bd, _), g in zip(grey, got):
        assert np.array_equal(g, O.convert(img, ct, bd, 1)), (img.shape, ct, bd)


def test_decode_png_matches_cv2_goldens(ctx):
    g = np.load(GOLDEN)
    names = list(g["names"])
    pngs = [g[f"png_{i}"].tobytes() for i in range(len(names))]
    for i, out in enumerate(ctx.decode_png(pngs, 3)):
        assert np.array_equal(out, g[f"color_{i}"]), names[i]
    grey = [i for i in range(len(names)) if f"gray_{i}" in g]
    for i, out in zip(grey, ctx.decode_png([pngs[i] for i in grey], 1)):
        assert np.array_equal(out, g[f"gray_{i}"]), names[i]


def test_decode_png_refusals_name_frame_and_reason(ctx):
    good = O.encode(np.arange(64, dtype=np.uint8).reshape(8, 8), 0, 8)
    z = O.zstream(good)
    trunc = O.with_zstream(good, z[: len(z) // 2])
    bad_adler = O.with_zstream(good, z[:-1] + bytes([z[-1] ^ 1]))
    with pytest.raises(XivoError, match="frame 1: truncated deflate"):
        ctx.decode_png([good, trunc, good], 3)
    with pytest.raises(XivoError, match="frame 2: Adler-32"):
        ctx.decode_png([good, good, bad_adler], 3)
    with pytest.raises(XivoError, match="1-channel output"):
        ctx.decode_png([O.encode(np.zeros((2, 2, 3), np.uint8), 2, 8)], 1)
    assert np.array_equal(ctx.decode_png([good], 1)[0], np.arange(64, dtype=np.uint8).reshape(8, 8))  # the context still works


# ------------------------------------------------------------------------------------------------ pyxivo
def small_cfg():
    cfg = sim.load_cfg(os.path.join(CFG, "vio_640x480.json"))
    cfg["camera_cfg"].update(rows=240, cols=320, fx=137.5, fy=137.5, cx=160, cy=120)
    cfg["tracker_cfg"].update(num_features_min=60, num_features_max=80)
    return cfg


def encode_frame(img, seq, k):
    """a sequence-specific PNG form of a cv2.imread result: 8 / 16 bits, grey or RGB, level and filters vary"""
    rng = np.random.default_rng(1000 * seq + k)
    bd = 16 if seq % 2 else 8
    if img.ndim == 2:
        s = img.astype(np.uint16) << 8 | rng.integers(0, 256, img.shape).astype(np.uint16) if bd == 16 else img
        ct = 0
    else:
        s = img[..., ::-1]
        s = s.astype(np.uint16) << 8 | rng.integers(0, 256, s.shape).astype(np.uint16) if bd == 16 else s
        ct = 2
    return O.encode(s, ct, bd, filters=None if seq % 3 else 4, level=[1, 6, 9][seq % 3], seed=k)


def snapshot(b):
    return [(b.now(s), b.gsb(s), b.counters(s)) for s in range(b.n)]


def same(x, y):
    for (ta, ga, ca), (tb, gb, cb) in zip(x, y):
        assert ta == tb and np.array_equal(ga, gb) and ca == cb


@pytest.mark.parametrize("channels,tracker_only", [(1, False), (3, False), (1, True)])
def test_batch_visual_meas_png_is_bit_identical_to_arrays(channels, tracker_only):
    cfg = small_cfg()
    n = 8
    streams = [sim.image_stream(cfg, duration=1.0, seed=11 + s, channels=channels)[0] for s in range(n)]
    a = pyxivo.Batch(cfg, n_seq=n, max_groups=4, max_features=14, tracker_only=tracker_only)
    b = pyxivo.Batch(cfg, n_seq=n, max_groups=4, max_features=14, tracker_only=tracker_only)
    frames = 0
    for k, msgs in enumerate(zip(*streams)):
        kinds = {m[0] for m in msgs}
        assert len(kinds) == 1
        ts = [m[1] for m in msgs]
        if "imu" in kinds:
            g = np.array([m[2][0] for m in msgs])
            acc = np.array([m[2][1] for m in msgs])
            a.inertial_meas(ts, g, acc)
            b.inertial_meas(ts, g, acc)
            continue
        imgs = [m[2] for m in msgs]
        a.visual_meas(ts, imgs, tracker_only=tracker_only)
        b.visual_meas_png(ts, [encode_frame(im, s, k) for s, im in enumerate(imgs)], channels=channels, tracker_only=tracker_only)
        same(snapshot(a), snapshot(b))
        frames += 1
    assert frames >= 20
    assert np.array_equal(a.P(), b.P())
    a.close()
    b.close()


def test_estimator_visual_meas_path_over_asl_folder_of_16bit_pngs(tmp_path):
    """the scripts/pyxivo.py loop over a data.csv of 16-bit grey PNG files (TUM-VI 512_16 style)"""
    cfg = small_cfg()
    msgs, _ = sim.image_stream(cfg, duration=1.4, seed=5, channels=3)
    cam = tmp_path / "cam0" / "data"
    cam.mkdir(parents=True)
    rng = np.random.default_rng(0)
    ref = pyxivo.Estimator(cfg, max_groups=4, max_features=14)
    est = pyxivo.Estimator(cfg, max_groups=4, max_features=14)
    lines, n = [], 0
    for kind, ts, p in msgs:
        if kind == "imu":
            ref.InertialMeas(ts, *p[0], *p[1])
            est.InertialMeas(ts, *p[0], *p[1])
            continue
        grey = p[..., 0]
        path = str(cam / f"{ts}.png")
        with open(path, "wb") as f:
            f.write(O.encode(grey.astype(np.uint16) << 8 | rng.integers(0, 256, grey.shape).astype(np.uint16), 0, 16))
        lines.append(f"{ts},{ts}.png")
        ref.VisualMeas(ts, np.repeat(grey[..., None], 3, axis=2))  # cv::imread(path) of a grey file: grey in all three channels
        est.VisualMeas(ts, path)
        assert est.now() == ref.now() and np.array_equal(est.gsb(), ref.gsb())
        n += 1
    assert n >= 30
    assert np.array_equal(est.P(), ref.P())
    pgm = tmp_path / "frame.pgm"
    pgm.write_bytes(b"P5 4 4 255\n" + bytes(16))
    with pytest.raises(XivoError, match="bad signature"):
        est.VisualMeas(msgs[-1][1] + 1, str(pgm))


def test_refused_batch_calls_leave_every_sequence_untouched():
    cfg = small_cfg()
    n = 4
    streams = [sim.image_stream(cfg, duration=0.8, seed=21 + s, channels=1)[0] for s in range(n)]
    a = pyxivo.Batch(cfg, n_seq=n, max_groups=4, max_features=14)
    b = pyxivo.Batch(cfg, n_seq=n, max_groups=4, max_features=14)
    pal = O.SIG + O.chunk(b"IHDR", bytes.fromhex("0000000400000004") + bytes([8, 3, 0, 0, 0])) + O.chunk(b"IEND", b"")
    refused, j = 0, 0
    for k, msgs in enumerate(zip(*streams)):
        ts = [m[1] for m in msgs]
        if msgs[0][0] == "imu":
            g, acc = np.array([m[2][0] for m in msgs]), np.array([m[2][1] for m in msgs])
            a.inertial_meas(ts, g, acc)
            b.inertial_meas(ts, g, acc)
            continue
        pngs = [O.encode(m[2], 0, 8, seed=k) for m in msgs]
        j += 1
        if j % 3 == 1:
            bad = list(pngs)
            z = O.zstream(pngs[1])
            kind = (j // 3) % 4
            if kind == 0:
                bad[1] = O.with_zstream(pngs[1], z[: len(z) // 2])
                why = "frame 1: truncated deflate"
            elif kind == 1:
                bad[1] = O.with_zstream(pngs[1], z[:-1] + bytes([z[-1] ^ 4]))
                why = "frame 1: Adler-32"
            elif kind == 2:
                bad[1] = pal
                why = "frame 1: palette"
            else:
                bad[1] = O.encode(msgs[1][2][:-1], 0, 8)
                why = "frame 1 is 239 x 320, frame 0 is 240 x 320"
            with pytest.raises(XivoError, match=why):
                b.visual_meas_png(ts, bad, channels=1)
            refused += 1
        a.visual_meas(ts, [m[2] for m in msgs])
        b.visual_meas_png(ts, pngs, channels=1)
        same(snapshot(a), snapshot(b))
    assert refused >= 3
    assert np.array_equal(a.P(), b.P())
    a.close()
    b.close()
