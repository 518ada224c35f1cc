"""numpy restatement of the per-pixel work of the reference's optical_flow_homography (getimage / infer / resize_flow): the registration
cv2.warpPerspective(frame2, H_BA, (W, H)) of an 8-bit BGR frame, cv::invert's closed-form 3 x 3 inverse, the un-registration through
np.linalg.inv(H_BA).dot, and cv2.resize(float64 flow, INTER_CUBIC) times (w / W, h / H).  The kernels of rcvd_flowreg.cuh follow it op
for op; tests/test_flow_register.py pins it against OpenCV and numpy."""
import numpy as np

TAB = 32            # INTER_TAB_SIZE: 5 fractional bits per source coordinate
COEF_BITS = 15      # INTER_REMAP_COEF_BITS


def cv_invert3(M):
    """cv::invert(M, DECOMP_LU) of a 3 x 3 double matrix (its closed form for n = 3): cofactors times 1 / det, det expanded along row 0;
    a zero det gives the zero matrix."""
    m = np.asarray(M, np.float64).reshape(3, 3)
    det = (m[0, 0] * (m[1, 1] * m[2, 2] - m[1, 2] * m[2, 1]) - m[0, 1] * (m[1, 0] * m[2, 2] - m[1, 2] * m[2, 0])
           + m[0, 2] * (m[1, 0] * m[2, 1] - m[1, 1] * m[2, 0]))
    if det == 0:
        return np.zeros((3, 3))
    d = 1.0 / det
    t = [(m[1, 1] * m[2, 2] - m[1, 2] * m[2, 1]) * d, (m[0, 2] * m[2, 1] - m[0, 1] * m[2, 2]) * d, (m[0, 1] * m[1, 2] - m[0, 2] * m[1, 1]) * d,
         (m[1, 2] * m[2, 0] - m[1, 0] * m[2, 2]) * d, (m[0, 0] * m[2, 2] - m[0, 2] * m[2, 0]) * d, (m[0, 2] * m[1, 0] - m[0, 0] * m[1, 2]) * d,
         (m[1, 0] * m[2, 1] - m[1, 1] * m[2, 0]) * d, (m[0, 1] * m[2, 0] - m[0, 0] * m[2, 1]) * d, (m[0, 0] * m[1, 1] - m[0, 1] * m[1, 0]) * d]
    return np.array(t, np.float64).reshape(3, 3)


def warp_weights():
    """The [TAB * TAB, 4] int32 bilinear weights of fractional index fy * TAB + fx, taps (0,0), (1,0), (0,1), (1,1) (x first): the float
    products (1 - fx/32 or fx/32)(1 - fy/32 or fy/32) times 2^15, all exact, so they sum to 2^15 and OpenCV's sum fix-up never applies."""
    f = np.arange(TAB)
    fy, fx = np.meshgrid(f, f, indexing="ij")
    w = np.stack([(TAB - fx) * (TAB - fy), fx * (TAB - fy), (TAB - fx) * fy, fx * fy], -1).reshape(-1, 4)
    return (w * ((1 << COEF_BITS) // (TAB * TAB))).astype(np.int32)


def warp_block_width(W, H):
    """The width of warpPerspective's pixel blocks: bh = min(16, H), bw = min(1024 // bh, W).  Each block row starts its coordinates at
    the block's first column x0 and adds M[0] (x - x0), so the block width is part of the arithmetic."""
    return min(1024 // min(16, H), W)


def warp_maps(Minv, W, H):
    """(sx, sy, alpha) int32 [H, W]: warpPerspective's fixed-point source map for the inverse matrix Minv (what cv2 uses after inverting
    H_BA), as its row loop computes it in double without FMA:
      X0 = (M0 x0 + M1 y) + M2, likewise Y0 and W0, at the block's first column x0;
      w = W0 + M6 (x - x0);  w = 32 / w, or 0 when w == 0;
      X = clamp((X0 + M0 (x - x0)) w, INT_MIN, INT_MAX) rounded half to even, likewise Y;
      sx = X >> 5, sy = Y >> 5 (saturated to int16), alpha = (Y & 31) * 32 + (X & 31)."""
    M = np.asarray(Minv, np.float64).reshape(9)
    bw = warp_block_width(W, H)
    x = np.arange(W)
    x0 = (x // bw * bw).astype(np.float64)[None, :]
    x1 = (x % bw).astype(np.float64)[None, :]
    y = np.arange(H, dtype=np.float64)[:, None]
    X0 = M[0] * x0 + M[1] * y + M[2]
    Y0 = M[3] * x0 + M[4] * y + M[5]
    W0 = M[6] * x0 + M[7] * y + M[8]
    w = W0 + M[6] * x1
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        w = np.where(w != 0, TAB / np.where(w != 0, w, 1.0), 0.0)
        X = np.clip((X0 + M[0] * x1) * w, -2.0 ** 31, 2.0 ** 31 - 1)
        Y = np.clip((Y0 + M[3] * x1) * w, -2.0 ** 31, 2.0 ** 31 - 1)
    Xi = np.rint(X).astype(np.int64)
    Yi = np.rint(Y).astype(np.int64)
    sx = np.clip(Xi >> 5, -32768, 32767).astype(np.int32)
    sy = np.clip(Yi >> 5, -32768, 32767).astype(np.int32)
    alpha = ((Yi & 31) * TAB + (Xi & 31)).astype(np.int32)
    return sx, sy, alpha


def warp_perspective(src, H_BA):
    """cv2.warpPerspective(src, H_BA, (W, H)) of a u8 [H, W, 3] image, INTER_LINEAR, BORDER_CONSTANT 0: the map of warp_maps for
    cv_invert3(H_BA), then per channel (sum of weight * tap + 2^14) >> 15 with the taps outside the image read as 0."""
    src = np.asarray(src, np.uint8)
    H, W = src.shape[:2]
    sx, sy, alpha = warp_maps(cv_invert3(H_BA), W, H)
    wt = warp_weights()[alpha]
    acc = np.full((H, W, 3), 1 << (COEF_BITS - 1), np.int64)
    for k, (dx, dy) in enumerate(((0, 0), (1, 0), (0, 1), (1, 1))):
        tx, ty = sx + dx, sy + dy
        inside = (tx >= 0) & (tx < W) & (ty >= 0) & (ty < H)
        v = src[np.clip(ty, 0, H - 1), np.clip(tx, 0, W - 1)].astype(np.int64) * inside[..., None]
        acc += v * wt[..., k:k + 1]
    return np.clip(acc >> COEF_BITS, 0, 255).astype(np.uint8)


def _two_sum(a, b):
    s = a + b
    bb = s - a
    return s, (a - (s - bb)) + (b - bb)


def _split(a):
    c = 134217729.0 * a     # 2^27 + 1
    hi = c - (c - a)
    return hi, a - hi


def _two_prod(a, b):
    p = a * b
    ah, al = _split(a)
    bh, bl = _split(b)
    return p, ((ah * bh - p) + ah * bl + al * bh) + al * bl


def fma(a, b, c):
    """Correctly rounded a * b + c in float64 arrays (Boldo and Melquiond's emulation: exact product and sum, the low parts added with
    round-to-odd, then one rounding).  Valid away from overflow and underflow, which the coordinates here never reach."""
    a, b, c = np.broadcast_arrays(np.asarray(a, np.float64), np.asarray(b, np.float64), np.asarray(c, np.float64))
    uh, ul = _two_prod(a, b)
    th, tl = _two_sum(c, uh)
    v, e = _two_sum(tl, ul)
    even = (v.view(np.int64) & 1) == 0
    fix = (e != 0) & even
    v = np.where(fix, np.nextafter(v, np.where(e > 0, np.inf, -np.inf)), v)
    return th + v


def unregister(flow, Hinv, order="fma"):
    """infer's un-registration: fxx = fx + u and fyy = fy + v in float32, then Hinv.dot([fxx; fyy; 1]) in float64, each row as
    OpenBLAS' dgemm computes it on x86-64 (order "fma": fma(h2, 1, fma(h1, y, h0 x))) or as the plain sum (order "plain":
    (h0 x + h1 y) + h2), then x / z - fx and y / z - fy.  flow float32 [H, W, 2]; returns float64 [H, W, 2]."""
    flow = np.asarray(flow, np.float32)
    H, W = flow.shape[:2]
    fy, fx = np.mgrid[0:H, 0:W].astype(np.float32)
    X = (fx + flow[..., 0]).astype(np.float64)
    Y = (fy + flow[..., 1]).astype(np.float64)
    h = np.asarray(Hinv, np.float64).reshape(3, 3)
    rows = []
    for r in range(3):
        if order == "fma":
            rows.append(fma(h[r, 2], 1.0, fma(h[r, 1], Y, h[r, 0] * X)))
        else:
            rows.append((h[r, 0] * X + h[r, 1] * Y) + h[r, 2])
    with np.errstate(divide="ignore", invalid="ignore"):
        return np.stack([rows[0] / rows[2] - fx, rows[1] / rows[2] - fy], -1)


def cubic_coeffs(f):
    """interpolateCubic in float32 (A = -0.75, no FMA), the last coefficient 1 - c0 - c1 - c2."""
    f = np.asarray(f, np.float32)
    A = np.float32(-0.75)
    one = np.float32(1)
    x1 = f + one
    c0 = ((A * x1 - np.float32(5) * A) * x1 + np.float32(8) * A) * x1 - np.float32(4) * A
    c1 = ((A + np.float32(2)) * f - (A + np.float32(3))) * f * f + one
    g = one - f
    c2 = ((A + np.float32(2)) * g - (A + np.float32(3))) * g * g + one
    c3 = one - c0 - c1 - c2
    return np.stack([c0, c1, c2, c3], -1)


def cubic_axis(n, m):
    """(first tap, float32 [m, 4] coefficients, interior) of cv2.resize's INTER_CUBIC for n source samples -> m outputs: the scale
    1 / (m / n) in double, f = float32((d + 0.5) s - 0.5), s0 = floor(f), f -= s0 in float32; taps s0 - 1 .. s0 + 2, clamped to
    [0, n - 1].  interior: all four taps inside (the horizontal pass sums border columns from 0, so a -0 sum becomes +0 there)."""
    s = 1.0 / (m / n)
    f = ((np.arange(m) + 0.5) * s - 0.5).astype(np.float32)
    s0 = np.floor(f).astype(np.int64)
    f = f - s0.astype(np.float32)
    return s0, cubic_coeffs(f), (s0 >= 1) & (s0 + 2 <= n - 1)


def resize_cubic(img, w, h):
    """cv2.resize(img, (w, h), interpolation=INTER_CUBIC) of a float64 [H, W, C] image: a copy when the size is unchanged; otherwise
    the horizontal pass ((p0 + p1) + p2) + p3 in float64 (0 + p0 + ... at border columns), then the vertical pass likewise over the
    clamped rows."""
    img = np.asarray(img, np.float64)
    H, W = img.shape[:2]
    if (w, h) == (W, H):
        return img.copy()
    xs, ax, xin = cubic_axis(W, w)
    ys, ay, _ = cubic_axis(H, h)
    ax = ax.astype(np.float64)
    ay = ay.astype(np.float64)
    cols = [img[:, np.clip(xs + k - 1, 0, W - 1)] * ax[None, :, k, None] for k in range(4)]
    border = ((0.0 + cols[0]) + cols[1]) + cols[2] + cols[3]
    inner = ((cols[0] + cols[1]) + cols[2]) + cols[3]
    hz = np.where(xin[None, :, None], inner, border)
    rows = [hz[np.clip(ys + k - 1, 0, H - 1)] * ay[:, k, None, None] for k in range(4)]
    return ((rows[0] + rows[1]) + rows[2]) + rows[3]


def resize_flow(flow, w, h):
    """resize_flow(flow, (w, h)): resize_cubic, then times (w / W, h / H) in float64."""
    H, W = flow.shape[:2]
    return resize_cubic(flow, w, h) * np.array([w / float(W), h / float(H)])


def flow_raw_values(flow, Hinv, w, h, order="fma"):
    """The float32 [h, w, 2] values of flow/flow_i_j.raw from the model's float32 flow and np.linalg.inv(H_BA)."""
    return resize_flow(unregister(flow, Hinv, order), w, h).astype(np.float32)
