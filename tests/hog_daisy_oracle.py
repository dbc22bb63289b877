"""NumPy restatement of the reference's HOG and DAISY descriptors (K/nodes/images/HogExtractor.scala,
K/nodes/images/DaisyExtractor.scala and ImageUtils.conv2D), in the reference's operation order (DESIGN.md section 19).

Images are img[x, y, c] with x the Image's row (xDim = height) and, for HOG, channels in BGR order as ImageUtils.loadImage
delivers them.  NumPy never fuses a multiply into an add, and np.add.at adds its (index, value) pairs in the order given, so
the fp32 histogram below receives its addends in the reference's pixel order (x outer, y inner)."""
import math

import numpy as np

F32, F64 = np.float32, np.float64

# ------------------------------------------------------------------------------------------------------------------------ HOG
HOG_UU = (1.0000, 0.9397, 0.7660, 0.500, 0.1736, -0.1736, -0.5000, -0.7660, -0.9397)
HOG_VV = (0.0000, 0.3420, 0.6428, 0.8660, 0.9848, 0.9848, 0.8660, 0.6428, 0.3420)
HOG_EPS = 0.0001
HOG_FEATURES = 32


def hog_cells(x_dim: int, y_dim: int, bin_: int):
    """(nX, nY): Scala's math.round(dim / bin), i.e. floor(v + 0.5)."""
    return int(math.floor(x_dim / bin_ + 0.5)), int(math.floor(y_dim / bin_ + 0.5))


def hog_rows(x_dim: int, y_dim: int, bin_: int) -> int:
    """Rows of the feature matrix: the interior cells (nX - 2)(nY - 2), zero when either side has fewer than 3 cells."""
    nx, ny = hog_cells(x_dim, y_dim, bin_)
    return max(nx - 2, 0) * max(ny - 2, 0)


def hog_out_of_image(x_dim: int, y_dim: int, channels: int, bin_: int) -> bool:
    """True where the reference throws: the pixel loop reads the flat index c + x C + y C xDim of the channel-major image without
    clamping, and its largest read is channel 2 at (nX bin - 2, nY bin - 1)."""
    nx, ny = hog_cells(x_dim, y_dim, bin_)
    vx, vy = nx * bin_, ny * bin_
    if vx < 3 or vy < 3:
        return False
    return 2 + (vx - 2) * channels + (vy - 1) * channels * x_dim >= channels * x_dim * y_dim


def hog_extract(img: np.ndarray, bin_: int) -> np.ndarray:
    """HogExtractor(bin).apply on img[x, y, 3] (fp64 values, already / 255.0 when PixelScaler precedes it).  Returns the reference's
    ((nX - 2)(nY - 2) x 32) fp32 matrix, row y + x (nY - 2)."""
    img = np.asarray(img, dtype=F64)
    x_dim, y_dim, ch = img.shape
    if ch != 3:
        raise ValueError("HogExtractor reads channels 2, 1 and 0")
    if hog_out_of_image(x_dim, y_dim, ch, bin_):
        raise ValueError("HogExtractor: the pixel loop reads past the end of the image")
    nx, ny = hog_cells(x_dim, y_dim, bin_)
    flat = np.transpose(img, (1, 0, 2)).ravel()          # c + x C + y C xDim, the reference's unclamped reads wrap in it
    hist = np.zeros(18 * nx * ny, dtype=F32)
    xs, ys = np.arange(1, nx * bin_ - 1), np.arange(1, ny * bin_ - 1)
    if xs.size and ys.size:
        X, Y = (a.ravel() for a in np.meshgrid(xs, ys, indexing="ij"))   # x outer, y inner

        def get(x, y, c):
            return flat[c + x * ch + y * ch * x_dim]

        best = np.full(X.shape, -np.inf)
        bdx, bdy = np.zeros(X.shape), np.zeros(X.shape)
        for c in (2, 1, 0):
            dx = get(X + 1, Y, c) - get(X - 1, Y, c)
            dy = get(X, Y + 1, c) - get(X, Y - 1, c)
            m2 = dx * dx + dy * dy
            take = m2 > best
            best = np.where(take, m2, best)
            bdx, bdy = np.where(take, dx, bdx), np.where(take, dy, bdy)
        mag = np.sqrt(best)
        bdot = np.zeros(X.shape)
        ori = np.zeros(X.shape, dtype=np.int64)
        for o in range(9):
            dot = HOG_UU[o] * bdy + HOG_VV[o] * bdx
            pos = dot > bdot
            neg = ~pos & (-dot > bdot)
            ori = np.where(pos, o, np.where(neg, o + 9, ori))
            bdot = np.where(pos, dot, np.where(neg, -dot, bdot))
        yp = (Y + 0.5) / bin_ - 0.5
        xp = (X + 0.5) / bin_ - 0.5
        iyp, ixp = np.floor(yp).astype(np.int64), np.floor(xp).astype(np.int64)
        vy0, vx0 = yp - iyp, xp - ixp
        vy1, vx1 = 1.0 - vy0, 1.0 - vx0
        base = ori * nx * ny
        idx = np.stack([ixp + iyp * nx, ixp + (iyp + 1) * nx, ixp + 1 + iyp * nx, ixp + 1 + (iyp + 1) * nx], 1) + base[:, None]
        val = np.stack([vy1 * vx1 * mag, vy0 * vx1 * mag, vy1 * vx0 * mag, vy0 * vx0 * mag], 1).astype(F32)
        ok = np.stack([(iyp >= 0) & (ixp >= 0), (iyp + 1 < ny) & (ixp >= 0),
                       (iyp >= 0) & (ixp + 1 < nx), (iyp + 1 < ny) & (ixp + 1 < nx)], 1)
        np.add.at(hist, idx[ok], val[ok])                 # row-major over (pixel, term): the reference's order
    h = hist.reshape(18, ny, nx)                          # h[o, y, x]
    norm = np.zeros((ny, nx), dtype=F32)
    for o in range(9):
        s = h[o] + h[o + 9]
        norm = norm + s * s
    fx, fy = max(nx - 2, 0), max(ny - 2, 0)
    out = np.zeros((fx * fy, HOG_FEATURES), dtype=F32)
    if fx == 0 or fy == 0:
        return out
    cx, cy = (a.ravel() for a in np.meshgrid(np.arange(fx), np.arange(fy), indexing="ij"))   # row y + x fy

    def block(x0, y0):     # 1 / sqrt(four fp32 norms added in fp32, then + 1e-4 in fp64)
        s = norm[y0, x0] + norm[y0, x0 + 1] + norm[y0 + 1, x0] + norm[y0 + 1, x0 + 1]
        return 1.0 / np.sqrt(s.astype(F64) + HOG_EPS)

    ns = [block(cx + 1, cy + 1), block(cx, cy + 1), block(cx + 1, cy), block(cx, cy)]
    t = [np.zeros(cx.shape) for _ in range(4)]
    for o in range(18):
        v = h[o, cy + 1, cx + 1].astype(F64)
        hs = [np.minimum(v * n, 0.2) for n in ns]
        out[:, o] = (0.5 * (hs[0] + hs[1] + hs[2] + hs[3])).astype(F32)
        for k in range(4):
            t[k] = t[k] + hs[k]
    for o in range(9):
        v = (h[o, cy + 1, cx + 1] + h[o + 9, cy + 1, cx + 1]).astype(F64)
        hs = [np.minimum(v * n, 0.2) for n in ns]
        out[:, 18 + o] = (0.5 * (hs[0] + hs[1] + hs[2] + hs[3])).astype(F32)
    for k in range(4):
        out[:, 27 + k] = (0.2357 * t[k]).astype(F32)
    return out


def breeze_sum_f32(m: np.ndarray) -> float:
    """sum(DenseMatrix[Float]) as Breeze takes it: sequentially in fp32 over the column-major storage."""
    m = np.asarray(m, dtype=F32)
    return float(np.cumsum(m.T.ravel(), dtype=F32)[-1]) if m.size else 0.0


# ---------------------------------------------------------------------------------------------------------------------- DAISY
CONV_THRESHOLD = 1e-6
FEATURE_THRESHOLD = 1e-8


def daisy_taps(Q: int, R: int):
    """Per layer q < Q the Gaussian taps exp(-n^2 / 2 D) / sqrt(2 pi D), n = -t..t, where D = sigma_{q+1}^2 - sigma_q^2,
    sigma_n = R n / 2Q, and t = ceil(sqrt(-2 D ln 1e-6 - D ln 2 pi D))."""
    sq = []
    for n in range(Q + 1):
        s = R * float(n) / (2 * Q)
        sq.append(s * s)
    taps = []
    for q in range(Q):
        d = sq[q + 1] - sq[q]
        t = int(math.ceil(math.sqrt(-2 * d * math.log(CONV_THRESHOLD) - d * math.log(2 * math.pi * d))))
        taps.append(np.array([math.exp(-(float(n) ** 2 / (2 * d))) / math.sqrt(2 * math.pi * d) for n in range(-t, t + 1)]))
    return taps


def daisy_offsets(T: int, Q: int, R: int):
    """(dx, dy) of ring sample (l, t) at index l T + t: round(r_l sin theta), round(r_l cos theta), r_l = R (1 + l) / Q and the
    reference's theta = 2 pi (t - 1) / T; round is floor(v + 0.5)."""
    out = []
    for l in range(Q):
        rad = R * (1 + float(l)) / Q
        for t in range(T):
            th = 2 * math.pi * (t - 1) / T
            out.append((int(math.floor(rad * math.sin(th) + 0.5)), int(math.floor(rad * math.cos(th) + 0.5))))
    return out


def daisy_keypoints(x_dim: int, y_dim: int, border: int, stride: int):
    """Keypoint coordinates along x and along y: border to dim - border - 1 by stride."""
    return list(range(border, x_dim - border, stride)), list(range(border, y_dim - border, stride))


def conv2d(img: np.ndarray, xf, yf) -> np.ndarray:
    """ImageUtils.conv2D on a one-channel img[x, y] (fp64): zero padding, 'same' size, low pad floor((len - 1) / 2), the filters
    reversed; a pass along x, then along y, each output an fp64 running sum from 0.0 over the taps in ascending order."""
    img = np.asarray(img, dtype=F64)
    X, Y = img.shape
    xf, yf = np.asarray(xf, dtype=F64), np.asarray(yf, dtype=F64)
    lx, ly = xf.size, yf.size
    px, py = (lx - 1) // 2, (ly - 1) // 2
    p = np.zeros((X + lx - 1, Y))
    p[px:px + X] = img
    mid = np.zeros((X, Y))
    for i in range(lx):
        mid = mid + p[i:i + X] * xf[lx - 1 - i]
    p = np.zeros((X, Y + ly - 1))
    p[:, py:py + Y] = mid
    res = np.zeros((X, Y))
    for j in range(ly):
        res = res + p[:, j:j + Y] * yf[ly - 1 - j]
    return res


def daisy_extract(gray: np.ndarray, T=8, Q=3, R=7, H=8, border=16, stride=4) -> np.ndarray:
    """DaisyExtractor(T, Q, R, H, border, stride).apply on a one-channel gray[x, y].  Returns one descriptor per ROW (the
    reference's columns): (nKP x H (T Q + 1)) fp32, keypoints x outer, y inner; columns: the centre at [0, H), ring sample (l, t) at
    H + t Q H + l H."""
    gray = np.asarray(gray, dtype=F64)
    X, Y = gray.shape
    kx, ky = daisy_keypoints(X, Y, border, stride)
    offs = daisy_offsets(T, Q, R)
    if kx and ky:
        for dx, dy in offs:
            if kx[0] + dx < 0 or kx[-1] + dx > X - 1 or ky[0] + dy < 0 or ky[-1] + dy > Y - 1:
                raise ValueError("DaisyExtractor: a ring sample leaves the image")
    taps = daisy_taps(Q, R)
    ix = conv2d(gray, [1.0, 0.0, -1.0], [1.0, 2.0, 1.0])
    iy = conv2d(gray, [1.0, 2.0, 1.0], [1.0, 0.0, -1.0])
    layers = [[None] * H for _ in range(Q)]
    for a in range(H):
        ang = 2 * math.pi * a / H
        v = np.maximum(math.cos(ang) * ix + math.sin(ang) * iy, 0.0)
        layers[0][a] = conv2d(v, taps[0], taps[0])
        for l in range(1, Q):
            layers[l][a] = conv2d(layers[l - 1][a], taps[l], taps[l])
    stack = [np.stack(layers[l], -1) for l in range(Q)]    # [x, y, h]
    F = H * (T * Q + 1)
    out = np.zeros((len(kx) * len(ky), F), dtype=F32)
    if not out.size:
        return out
    KX, KY = (a.ravel() for a in np.meshgrid(np.asarray(kx), np.asarray(ky), indexing="ij"))

    def normalized(v):      # v [nKP, H]: the fp64 norm summed in order; zero below 1e-8
        s = np.zeros(v.shape[0])
        for h in range(H):
            s = s + v[:, h] * v[:, h]
        n = np.sqrt(s)
        keep = n > FEATURE_THRESHOLD
        return np.where(keep[:, None], v / np.where(keep, n, 1.0)[:, None], 0.0).astype(F32)

    out[:, :H] = normalized(stack[0][KX, KY])
    for l in range(Q):
        for t in range(T):
            dx, dy = offs[l * T + t]
            c0 = H + t * Q * H + l * H
            out[:, c0:c0 + H] = normalized(stack[l][KX + dx, KY + dy])
    return out
