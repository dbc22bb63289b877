"""NumPy restatement of the reference's dense multi-scale SIFT (K/nodes/images/external/SIFTExtractor.scala, the JNI driver
VLFeat.cxx:37-201 and 256-261, and vlfeat 0.9.20's vl_imsmooth_f / vl_dsift_process with a flat window), plus PixelScaler and
GrayScaler (ImageUtils.scala:73-103, 115-130).

Every step after the gray conversion is fp32 in vlfeat's operation order with separate multiplies and adds (vlfeat's x86 build has
no fused multiply-add); NumPy's add.accumulate is sequential, so the running sums below add in the same order as vlfeat's loops.
vlfeat sees an Image transposed: the driver passes width = xDim and a float array with x fastest, so vlfeat's row index is the
Image's y and its column index the Image's x (DESIGN.md section 18).

Descriptors come back one per row (the reference stores them one per column), in vlfeat's order: scales in order, then frames
with vlfeat-y outer and vlfeat-x inner."""
import math

import numpy as np

F32 = np.float32
TWO_PI_F = F32(2 * math.pi)
QUARTER_PI_F = F32(math.pi / 4)
THREE_QUARTER_PI_F = F32(3 * math.pi / 4)
FLT_EPSILON = F32(np.finfo(np.float32).eps)
CONTRAST_THRESHOLD = F32(0.005)
NUM_BIN_T, NUM_BIN_XY = 8, 4


# --------------------------------------------------------------------------------------------------------------- image preparation
def pixel_scale(img: np.ndarray) -> np.ndarray:
    """PixelScaler: x / 255.0 in fp64."""
    return np.asarray(img, dtype=np.float64) / 255.0


def gray_scale(img: np.ndarray) -> np.ndarray:
    """GrayScaler on img[x, y, c] (fp64): 0.2989 R + 0.5870 G + 0.1140 B with B at channel 0 for three channels, left to right;
    sqrt(sum_c v^2 / C) otherwise. Returns [x, y] fp64."""
    img = np.asarray(img, dtype=np.float64)
    if img.shape[2] == 3:
        return 0.2989 * img[:, :, 2] + 0.5870 * img[:, :, 1] + 0.1140 * img[:, :, 0]
    acc = np.zeros(img.shape[:2])
    for c in range(img.shape[2]):
        acc = acc + img[:, :, c] * img[:, :, c]
    return np.sqrt(acc / img.shape[2])


def gray_f32(rgb_hwc: np.ndarray) -> np.ndarray:
    """An 8-bit RGB file through ImageUtils.loadImage (BGR, x = row), PixelScaler and GrayScaler, rounded once to fp32 as
    getSingleChannelAsFloatArray does: [x, y] fp32."""
    bgr = np.asarray(rgb_hwc)[:, :, ::-1].astype(np.float64)
    return gray_scale(pixel_scale(bgr)).astype(F32)


# --------------------------------------------------------------------------------------------------------------------- geometry
def scale_geometry(x_dim: int, y_dim: int, step: int, bin_: int, scales: int, scale_step: int):
    """Per scale: (bin_s, step_s, min, frames along vlfeat x (= Image x), frames along vlfeat y (= Image y)).
    Bounds are (off, off, W - 1, H - 1) with off = 1 + 2 scales - 3 s; vl_dsift_set_bounds clamps a negative minimum to 0."""
    out = []
    for s in range(scales):
        b, st = bin_ + 2 * s, step + s * scale_step
        lo = max(1 + 2 * scales - 3 * s, 0)
        n = []
        for dim in (x_dim, y_dim):
            rng = (dim - 1) - lo - (NUM_BIN_XY - 1) * b
            n.append(rng // st + 1 if rng >= 0 else 0)
        out.append((b, st, lo, n[0], n[1]))
    return out


def keypoint_counts(x_dim, y_dim, step=3, bin_=4, scales=4, scale_step=1):
    return [nx * ny for (_, _, _, nx, ny) in scale_geometry(x_dim, y_dim, step, bin_, scales, scale_step)]


# -------------------------------------------------------------------------------------------------------------------- filters
def gaussian_filter(sigma: float) -> np.ndarray:
    """vl_imsmooth's kernel: radius ceil(4 sigma), taps exp(-x^2 / 2 sigma^2) in fp64 stored as fp32, divided by their fp32 sum
    taken in tap order. (A ceil(3 sigma) radius matches feats128 measurably worse: DESIGN.md section 18.)"""
    width = int(math.ceil(sigma * 4.0))
    filt = np.empty(2 * width + 1, dtype=F32)
    mass = F32(0.0)
    for j in range(2 * width + 1):
        x = (j - width) / sigma
        filt[j] = F32(math.exp(-0.5 * x * x))
        mass = mass + filt[j]
    return filt / mass


def conv_col(img: np.ndarray, filt: np.ndarray) -> np.ndarray:
    """vl_imconvcol_f along axis 0 with continuity padding: dest[y] = sum over p = y - r .. y + r (ascending) of
    img[clamp(p)] * filt[p - y + r], accumulated in fp32 from 0."""
    H = img.shape[0]
    r = (len(filt) - 1) // 2
    idx = np.arange(H)
    acc = np.zeros_like(img)
    for k in range(-r, r + 1):
        src = img[np.clip(idx + k, 0, H - 1)]
        acc = acc + src * filt[k + r]
    return acc


def smooth(im: np.ndarray, sigma: float) -> np.ndarray:
    """vl_imsmooth_f: the column pass (along vlfeat y) then the row pass, with the same kernel."""
    f = gaussian_filter(sigma)
    return conv_col(conv_col(im, f).T, f).T.copy()


def conv_col_tri(img: np.ndarray, F: int) -> np.ndarray:
    """vl_imconvcoltri_f along axis 0 with continuity padding: the unit-area triangle max(F - |t|, 0) / F^2 from two running sums.
    Backward integral B (from the last sample, F copies of the first sample appended); box R[y] = B[y] - B[y + F] (the tail uses
    B[H - 1] (H - F - y)); forward integral C from y = -F; out[y] = (1 / F^2) (C[y] - C[y - F])."""
    H = img.shape[0]
    ext = np.concatenate([np.repeat(img[:1], F, axis=0), img], axis=0)          # index j <-> y = j - F
    B = np.add.accumulate(ext[::-1], axis=0)[::-1]
    R = np.empty_like(B)
    head = max(H - F, -F) + F                                                    # rows y < H - F use B[y + F]
    R[:head] = B[:head] - B[F:F + head]
    ys = np.arange(head - F, H)
    R[head:] = B[head:] - B[H - 1 + F][None] * (H - F - ys).astype(F32)[:, None]
    C = np.add.accumulate(R, axis=0)
    scale = F32(1.0 / (float(F) * float(F)))
    return scale * (C[F:] - C[:H])


def bin_window_mean(bin_: int, index: int, window_size: float = 1.5) -> np.float32:
    """_vl_dsift_get_bin_window_mean: mean of exp(-z^2 / 2), z = (x - delta) / (bin window_size), over x in [-bin + 1, bin - 1],
    delta = bin (index - 1.5); the exp in fp64, the sum in fp32."""
    delta = F32(bin_) * (F32(index) - F32(0.5) * F32(NUM_BIN_XY - 1))
    sigma = F32(bin_) * F32(window_size)
    acc = F32(0.0)
    for x in range(-bin_ + 1, bin_):
        z = (F32(x) - delta) / sigma
        acc = F32(float(acc) + math.exp(float(F32(-0.5) * z * z)))
    return acc / F32(2 * bin_ - 1)


def bin_weights(bin_: int) -> np.ndarray:
    """w[by, bx] = (wx bin) (wy bin): the window mean times the bin size (the triangle is unit-area, SIFT wants unit height)."""
    w = [bin_window_mean(bin_, i) * F32(bin_) for i in range(NUM_BIN_XY)]
    return np.array([[w[bx] * w[by] for bx in range(NUM_BIN_XY)] for by in range(NUM_BIN_XY)], dtype=F32)


# ------------------------------------------------------------------------------------------------------------------ fast math
def fast_sqrt(x: np.ndarray) -> np.ndarray:
    """vl_fast_sqrt_f: x * resqrt(x) with the 0x5f3759df seed and two Newton steps; 0 below 1e-8 (a double literal)."""
    x = np.asarray(x, dtype=F32)
    xhalf = F32(0.5) * x
    y = (np.int32(0x5f3759df) - (x.view(np.int32) >> 1)).view(F32)
    y = y * (F32(1.5) - xhalf * y * y)
    y = y * (F32(1.5) - xhalf * y * y)
    return np.where(x.astype(np.float64) < 1e-8, F32(0), x * y).astype(F32)


def fast_atan2(y: np.ndarray, x: np.ndarray) -> np.ndarray:
    """vl_fast_atan2_f (c3 = 0.1821, c1 = 0.9675)."""
    abs_y = np.abs(y) + FLT_EPSILON
    pos = x >= 0
    num = np.where(pos, x - abs_y, x + abs_y)
    den = np.where(pos, x + abs_y, abs_y - x)
    r = num / den
    angle = np.where(pos, QUARTER_PI_F, THREE_QUARTER_PI_F)
    angle = angle + (F32(0.1821) * r * r - F32(0.9675)) * r
    return np.where(y < 0, -angle, angle).astype(F32)


# -------------------------------------------------------------------------------------------------------------------- dsift
def orientation_planes(im: np.ndarray) -> np.ndarray:
    """vl_dsift_process's gradient loop on im[vy, vx]: central differences inside, one-sided at the borders; the magnitude split
    linearly between the two nearest of 8 orientation bins. Returns [8, H, W]."""
    H, W = im.shape
    gy = np.empty_like(im)
    gx = np.empty_like(im)
    if H > 1:
        gy[1:-1] = F32(0.5) * (im[2:] - im[:-2])
        gy[0] = im[1] - im[0]
        gy[-1] = im[-1] - im[-2]
    else:
        gy[:] = 0
    if W > 1:
        gx[:, 1:-1] = F32(0.5) * (im[:, 2:] - im[:, :-2])
        gx[:, 0] = im[:, 1] - im[:, 0]
        gx[:, -1] = im[:, -1] - im[:, -2]
    else:
        gx[:] = 0
    angle = fast_atan2(gy, gx)
    mod = fast_sqrt(gx * gx + gy * gy)
    a = np.where(angle > TWO_PI_F, angle - TWO_PI_F, angle)
    a = np.where(a < F32(0), a + TWO_PI_F, a)
    nt = (a.astype(np.float64) * (NUM_BIN_T / (2 * math.pi))).astype(F32)
    bint = np.floor(nt).astype(np.int32)
    rbint = nt - bint.astype(F32)
    planes = np.zeros((NUM_BIN_T, H, W), dtype=F32)
    lo, hi = bint % NUM_BIN_T, (bint + 1) % NUM_BIN_T
    v_lo, v_hi = (F32(1) - rbint) * mod, rbint * mod
    for t in range(NUM_BIN_T):
        planes[t] = np.where(lo == t, v_lo, planes[t])
        planes[t] = np.where(hi == t, v_hi, planes[t])
    return planes


def _normalize(d: np.ndarray) -> np.ndarray:
    acc = np.zeros(d.shape[0], dtype=F32)
    for i in range(d.shape[1]):
        acc = acc + d[:, i] * d[:, i]
    return d / (fast_sqrt(acc) + FLT_EPSILON)[:, None]


def transpose_perm() -> np.ndarray:
    """vl_dsift_transpose_descriptor(., 8, 4, 4) as a gather: out[j] = raw[perm[j]]."""
    perm = np.empty(128, dtype=np.int64)
    for y in range(NUM_BIN_XY):
        for x in range(NUM_BIN_XY):
            off, off_t = NUM_BIN_T * (x + y * NUM_BIN_XY), NUM_BIN_T * (y + x * NUM_BIN_XY)
            for t in range(NUM_BIN_T):
                perm[off_t + (NUM_BIN_T // 4 - t + NUM_BIN_T) % NUM_BIN_T] = off + t
    return perm


def dsift_scale(im: np.ndarray, b: int, st: int, lo: int, nfx: int, nfy: int):
    """One scale on the smoothed image im[vy, vx]: raw descriptors [n, 128] (layout t + 8 bx + 32 by, frames vy-outer) and the
    keypoint mass (descriptor sum / (3 b + 1)^2), before normalisation."""
    planes = orientation_planes(im)
    n = nfx * nfy
    raw = np.zeros((n, 128), dtype=F32)
    if n == 0:
        return raw, np.zeros(0, dtype=F32)
    w = bin_weights(b)
    fy = lo + st * np.arange(nfy)
    fx = lo + st * np.arange(nfx)
    for t in range(NUM_BIN_T):
        tri = conv_col_tri(conv_col_tri(planes[t], b).T, b).T
        for by in range(NUM_BIN_XY):
            for bx in range(NUM_BIN_XY):
                v = tri[np.ix_(fy + by * b, fx + bx * b)].reshape(-1)
                raw[:, t + NUM_BIN_T * bx + NUM_BIN_T * NUM_BIN_XY * by] = w[by, bx] * v
    mass = np.zeros(n, dtype=F32)
    for i in range(128):
        mass = mass + raw[:, i]
    mass = mass / F32((3 * b + 1) * (3 * b + 1))
    return raw, mass


def finish(raw: np.ndarray, mass: np.ndarray) -> np.ndarray:
    """Normalise, clamp at 0.2, normalise; zero the keypoints with mass < 0.005; transpose; min((unsigned)(512 v), 255)."""
    d = _normalize(raw)
    d = np.minimum(d, F32(0.2))
    d = _normalize(d)
    d[mass < CONTRAST_THRESHOLD] = 0
    d = d[:, transpose_perm()]
    return np.minimum(np.floor(F32(512) * d), F32(255)).astype(F32)


def sift_extract(gray_xy: np.ndarray, step: int = 3, bin_: int = 4, scales: int = 4, scale_step: int = 1, with_mass: bool = False):
    """SIFTExtractor(step, bin, scales, scaleStep) on a gray Image gray_xy[x, y] (fp32): [nKP, 128] fp32 integer values in
    [0, 255], and with_mass=True also the fp32 keypoint mass the contrast threshold compares."""
    g = np.asarray(gray_xy, dtype=F32)
    X, Y = g.shape
    im = np.ascontiguousarray(g.T)                                               # vlfeat [vy, vx] = Image [x = vx, y = vy]
    descs, masses = [], []
    for (b, st, lo, nfx, nfy) in scale_geometry(X, Y, step, bin_, scales, scale_step):
        sm = smooth(im, b / 6.0)
        raw, mass = dsift_scale(sm, b, st, lo, nfx, nfy)
        descs.append(finish(raw, mass))
        masses.append(mass)
    D = np.concatenate(descs, 0) if descs else np.zeros((0, 128), F32)
    M = np.concatenate(masses, 0) if masses else np.zeros(0, F32)
    return (D, M) if with_mass else D
