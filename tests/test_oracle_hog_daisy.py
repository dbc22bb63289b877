"""The NumPy restatement of HogExtractor and DaisyExtractor (tests/hog_daisy_oracle.py) against the reference suites' MATLAB sums on
images/gantrycrane.png, against literal scalar transcriptions of the reference's loops, and its shapes and layouts."""
import math
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import hog_daisy_oracle as hd  # noqa: E402
import sift_oracle as so  # noqa: E402


def _bgr(golden_dir):
    """images/gantrycrane.png as ImageUtils.loadImage yields it: [x = row, y, c] with c in BGR order, fp64."""
    return np.load(os.path.join(golden_dir, "conv_gantrycrane.npz"))["rgb"][:, :, ::-1].astype(np.float64)


# ------------------------------------------------------------------------------------------------------------------------ HOG
def test_hog_matches_matlab_sums(golden_dir):
    """HogExtractorSuite: PixelScaler then HogExtractor(50) and (8); Breeze sums the (cells x 32) Float matrix in fp32, column by
    column, and the suite compares (ours - matlab) / ours to 1e-8 and 1e-4."""
    img = _bgr(golden_dir) / 255.0
    for bin_, matlab, tol in ((50, 59.2162514, 1e-8), (8, 4.5775269e+03, 1e-4)):
        F = hd.hog_extract(img, bin_)
        nx, ny = hd.hog_cells(264, 400, bin_)
        assert F.shape == ((nx - 2) * (ny - 2), 32) and F.dtype == np.float32
        ours = hd.breeze_sum_f32(F)
        assert abs((ours - matlab) / ours) < tol, (bin_, (ours - matlab) / ours)
        assert not F[:, 31].any()


def _hog_scalar(img, bin_):
    """HogExtractor.apply transcribed loop by loop (scatter into the fp32 histogram, unclamped flat reads) on a small image."""
    x_dim, y_dim, ch = img.shape
    flat = np.transpose(img, (1, 0, 2)).ravel()
    nx, ny = int(math.floor(x_dim / bin_ + 0.5)), int(math.floor(y_dim / bin_ + 0.5))
    hist = np.zeros(nx * ny * 18, dtype=np.float32)

    def get(x, y, c):
        return float(flat[c + x * ch + y * ch * x_dim])

    for x in range(1, nx * bin_ - 1):
        for y in range(1, ny * bin_ - 1):
            best, bdx, bdy = -math.inf, -math.inf, -math.inf
            for c in (2, 1, 0):
                dx = get(x + 1, y, c) - get(x - 1, y, c)
                dy = get(x, y + 1, c) - get(x, y - 1, c)
                if dx * dx + dy * dy > best:
                    best, bdx, bdy = dx * dx + dy * dy, dx, dy
            mag = math.sqrt(best)
            bdot, bo = 0.0, 0
            for o in range(9):
                dot = hd.HOG_UU[o] * bdy + hd.HOG_VV[o] * bdx
                if dot > bdot:
                    bo, bdot = o, dot
                elif -dot > bdot:
                    bo, bdot = o + 9, -dot
            yp, xp = (y + 0.5) / bin_ - 0.5, (x + 0.5) / bin_ - 0.5
            iyp, ixp = math.floor(yp), math.floor(xp)
            vy0, vx0 = yp - iyp, xp - ixp
            vy1, vx1 = 1.0 - vy0, 1.0 - vx0
            o = bo * nx * ny
            if iyp >= 0 and ixp >= 0:
                hist[ixp + iyp * nx + o] += np.float32(vy1 * vx1 * mag)
            if iyp + 1 < ny and ixp >= 0:
                hist[ixp + (iyp + 1) * nx + o] += np.float32(vy0 * vx1 * mag)
            if iyp >= 0 and ixp + 1 < nx:
                hist[ixp + 1 + iyp * nx + o] += np.float32(vy1 * vx0 * mag)
            if iyp + 1 < ny and ixp + 1 < nx:
                hist[ixp + 1 + (iyp + 1) * nx + o] += np.float32(vy0 * vx0 * mag)
    norm = np.zeros(nx * ny, dtype=np.float32)
    for o in range(9):
        for y in range(ny):
            for x in range(nx):
                s = hist[x + y * nx + o * nx * ny] + hist[x + y * nx + (o + 9) * nx * ny]
                norm[x + y * nx] += s * s
    fx, fy = max(nx - 2, 0), max(ny - 2, 0)
    out = np.zeros((fx * fy, 32), dtype=np.float32)
    for x in range(fx):
        for y in range(fy):
            def blk(off):
                return 1.0 / math.sqrt(float(norm[off] + norm[off + 1] + norm[off + nx] + norm[off + nx + 1]) + hd.HOG_EPS)
            n = [blk((y + 1) * nx + x + 1), blk((y + 1) * nx + x), blk(y * nx + x + 1), blk(y * nx + x)]
            t = [0.0] * 4
            base = (y + 1) * nx + x + 1
            for o in range(18):
                h = [min(float(hist[base + o * nx * ny]) * v, 0.2) for v in n]
                out[y + x * fy, o] = 0.5 * (h[0] + h[1] + h[2] + h[3])
                t = [a + b for a, b in zip(t, h)]
            for o in range(9):
                s = float(hist[base + o * nx * ny] + hist[base + (o + 9) * nx * ny])
                h = [min(s * v, 0.2) for v in n]
                out[y + x * fy, 18 + o] = 0.5 * (h[0] + h[1] + h[2] + h[3])
            for k in range(4):
                out[y + x * fy, 27 + k] = 0.2357 * t[k]
    return out


@pytest.mark.parametrize("shape,bin_", [((23, 17), 4), ((21, 31), 6), ((25, 26), 5), ((17, 12), 3)])
def test_hog_oracle_equals_scalar_transcription(shape, bin_):
    """Bit for bit, including shapes whose visible area nX bin passes xDim, so that reads wrap into the next column."""
    rng = np.random.default_rng(shape[0] * 100 + bin_)
    img = rng.integers(0, 256, size=shape + (3,)).astype(np.float64) / 255.0
    img[:, :, 1] = img[:, :, 2]              # equal channels: ties in the channel scan go to channel 2
    assert np.array_equal(hd.hog_extract(img, bin_), _hog_scalar(img, bin_))


def test_hog_wrap_and_rejection():
    # 23 rows at bin 4: round(5.75) = 6 cells, 24 visible rows; row 23 does not exist and the reads wrap into the next column
    assert hd.hog_cells(23, 17, 4) == (6, 4) and not hd.hog_out_of_image(23, 17, 3, 4)
    # a 500 x 375 VOC image (375 rows): at bin 4 only the rows round up (376 visible) and the last read is the image's last value;
    # at bin 8 the columns round up too (504 visible), which the reference cannot read
    assert hd.hog_cells(375, 500, 4) == (94, 125) and not hd.hog_out_of_image(375, 500, 3, 4)
    assert 2 + (376 - 2) * 3 + (500 - 1) * 3 * 375 == 3 * 375 * 500 - 1
    assert hd.hog_cells(375, 500, 8) == (47, 63) and hd.hog_out_of_image(375, 500, 3, 8)
    # both sides rounded up: the last read passes the end of the image, where the reference throws
    assert hd.hog_out_of_image(23, 23, 3, 4)
    with pytest.raises(ValueError):
        hd.hog_extract(np.zeros((23, 23, 3)), 4)
    # fewer than 3 cells along a side: no rows, and no read at all below 3 visible pixels
    assert hd.hog_extract(np.ones((9, 40, 3)), 4).shape == (0, 32)
    assert hd.hog_extract(np.ones((2, 2, 3)), 1).shape == (0, 32)
    assert hd.hog_rows(264, 400, 8) == 31 * 48


# ---------------------------------------------------------------------------------------------------------------------- DAISY
def test_daisy_matches_matlab_sums(golden_dir):
    """DaisyExtractorSuite: GrayScaler then DaisyExtractor(); the first keypoint's sum to 1e-5 and the full sum (fp64) to 1e-7,
    also with the gray image rounded to fp32 first, as the device takes it."""
    gray = so.gray_scale(_bgr(golden_dir))
    for g in (gray, gray.astype(np.float32)):
        D = hd.daisy_extract(g)
        assert D.shape == (5336, 200)
        first, total = 55.127217737738533, 3.240635661296463E5
        assert abs((D[0].astype(np.float64).sum() - first) / first) < 1e-5
        assert abs((D.astype(np.float64).sum() - total) / total) < 1e-7


def test_daisy_parameters_and_layout():
    assert [len(t) // 2 for t in hd.daisy_taps(3, 7)] == [6, 10, 13]
    offs = hd.daisy_offsets(8, 3, 7)
    # theta = 2 pi (t - 1) / T: ring sample t = 1 lies straight along +y, t = 0 one step before it
    assert offs[1] == (0, 2) and offs[0] == (-2, 2) and offs[2 * 8 + 1] == (0, 7)
    kx, ky = hd.daisy_keypoints(264, 400, 16, 4)
    assert (len(kx), len(ky)) == (58, 92) and kx[-1] == 244 and ky[-1] == 380
    rng = np.random.default_rng(4)
    gray = rng.random((45, 50))
    T, Q, R, H, border, stride = 5, 2, 6, 4, 7, 9
    D = hd.daisy_extract(gray, T, Q, R, H, border, stride)
    kx, ky = hd.daisy_keypoints(45, 50, border, stride)
    assert D.shape == (len(kx) * len(ky), H * (T * Q + 1))
    # the layers straight from the reference's definitions, and one keypoint's histograms in the reference's columns
    taps = hd.daisy_taps(Q, R)
    ix = hd.conv2d(gray, [1.0, 0.0, -1.0], [1.0, 2.0, 1.0])
    iy = hd.conv2d(gray, [1.0, 2.0, 1.0], [1.0, 0.0, -1.0])
    lay = [[None] * H for _ in range(Q)]
    for a in range(H):
        ang = 2 * math.pi * a / H
        lay[0][a] = hd.conv2d(np.maximum(math.cos(ang) * ix + math.sin(ang) * iy, 0.0), taps[0], taps[0])
        for l in range(1, Q):
            lay[l][a] = hd.conv2d(lay[l - 1][a], taps[l], taps[l])

    def unit(v):
        v = np.asarray(v)
        return (v / math.sqrt(sum(float(e) * float(e) for e in v))).astype(np.float32)

    for k in (0, 3, D.shape[0] - 1):
        x, y = kx[k // len(ky)], ky[k % len(ky)]
        assert np.array_equal(D[k, :H], unit([lay[0][a][x, y] for a in range(H)]))
        for l in range(Q):
            for t in range(T):
                th = 2 * math.pi * (t - 1) / T
                dx, dy = round_half_up(R * (1 + l) / Q * math.sin(th)), round_half_up(R * (1 + l) / Q * math.cos(th))
                col = H + t * Q * H + l * H
                assert np.array_equal(D[k, col:col + H], unit([lay[l][a][x + dx, y + dy] for a in range(H)]))
    # ring samples that leave the image are rejected
    with pytest.raises(ValueError):
        hd.daisy_extract(gray, border=5)
    assert hd.daisy_extract(rng.random((20, 20))).shape == (0, 200)   # no keypoint


def round_half_up(v):
    return int(math.floor(v + 0.5))


def test_conv2d_is_a_true_same_size_convolution():
    scipy_signal = pytest.importorskip("scipy.signal")
    rng = np.random.default_rng(1)
    img = rng.random((17, 23))
    xf, yf = rng.random(5), rng.random(4)
    ref = scipy_signal.convolve2d(img, np.outer(xf, yf), mode="full")[2:2 + 17, 2:2 + 23]
    assert np.abs(hd.conv2d(img, xf, yf) - ref).max() < 1e-12
