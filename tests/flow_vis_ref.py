"""CPU restatement of the flow visualisation (the reference's Flow.visualize_flow, flow.py:128-178): the Middlebury flow colouring
(utils/flowlib.py flow_to_image / compute_color / make_color_wheel), the masked composite (utils/visualization.py apply_mask, np.hstack /
np.vstack, cv2.imwrite's conversion to 8 bits) and the flow warp (flow.py warp_by_flow through utils/geometry.py sample), vectorised in
numpy with the dtypes the installed numpy (2.x, NEP 50 promotion) gives the reference's expressions:

  * rad = sqrt(u^2 + v^2) in float32 after zeroing unknown pixels (|u| or |v| > 1e7); maxrad = Python's max(-1, np.max(rad)), which
    is -1 when any rad is NaN (NaN > -1 is False), so that flow is divided by -1 + eps, i.e. negated; all-zero flows are divided by eps;
  * np.finfo(float).eps is a numpy float64, so u / (maxrad + eps) is float64, and atan2, fk, f, col are float64 as well (under numpy 1's
    value-based casting they were float32);
  * the 55-entry wheel, k1 = 56 wrapping to 1, col = 1 - rad (1 - col) inside the unit disc and 0.75 col outside, floor(255 col), NaN
    pixels (after the division) black, unknown pixels black;
  * apply_mask: 0.7 im + 0.3 (1 - (mask > 0)) [0, 255, 0]; 0.7 times a float32 colour stays float32, times a uint8 flow image is float64,
    and the stacked composite is float64; cv2.imwrite converts it with convertTo(CV_8U) (round half to even, saturate, and 0 where the
    rounded value leaves the int32 range or is NaN);
  * colour tiles are in the raw files' channel order and flow images in compute_color's RGB order: cv2.imwrite takes both as BGR.

The warp restates what torch's CUDA grid_sample kernel computes (the reference's device is CUDA when one is present): uv = pixel + flow and
grid = 2 uv / (W-1, H-1) - 1 in float32, source (g + 1) W / 2 - 1/2 clamped to [0, W-1] (NaN -> 0), the taps that lie in the image
weighted by products of distances.  Against torch's own grid_sample it agrees to a few float32 ulps, not to the bit (torch's result
depends on its kernel's FMA contraction): WARP_TOL states the bound."""
import numpy as np

f32 = np.float32
UNKNOWN_FLOW = 1e7
EPS = np.finfo(float).eps
WARP_TOL = 1e-5            # warp values within WARP_TOL (1 + |v|) of grid_sample's
# The Middlebury wheel: six hue segments of these lengths; in each, one channel stays at 255 while another ramps up or down in steps
# of floor(255 k / n): (length, channel at 255, ramping channel, ramps up).  Channels are R, G, B.
WHEEL_SEGMENTS = ((15, 0, 1, True), (6, 1, 0, False), (4, 1, 2, True), (11, 2, 1, False), (13, 2, 0, True), (6, 0, 2, False))


def color_wheel():
    """[55, 3] float64 wheel in RGB."""
    rows = []
    for n, full, ramp, up in WHEEL_SEGMENTS:
        seg = np.zeros((n, 3))
        seg[:, full] = 255
        r = np.floor(255 * np.arange(n) / n)
        seg[:, ramp] = r if up else 255 - r
        rows.append(seg)
    return np.concatenate(rows)


def flow_stats(flow):
    """(float32 max of rad over the non-NaN pixels after zeroing unknown ones, whether any rad is NaN, the unknown-pixel mask)."""
    u = flow[..., 0].astype(f32)
    v = flow[..., 1].astype(f32)
    unknown = (np.abs(u) > UNKNOWN_FLOW) | (np.abs(v) > UNKNOWN_FLOW)
    u = np.where(unknown, f32(0), u)
    v = np.where(unknown, f32(0), v)
    rad = np.sqrt(u * u + v * v)
    nan = np.isnan(rad)
    return (f32(rad[~nan].max()) if (~nan).any() else f32(0)), bool(nan.any()), unknown, u, v


def flow_image(flow, angle_ulps=0):
    """flowlib.flow_to_image: [H, W, 3] u8 in RGB order, plus (maxrad, has_nan) and the normalised float64 (u, v).  angle_ulps moves
    atan2's result by that many ulps (flow_image_margin)."""
    maxrad, has_nan, unknown, u, v = flow_stats(flow)
    d = (-1.0 if has_nan else float(maxrad)) + EPS          # max(-1, nan) is -1: the flow is negated, not normalised
    un = u.astype(np.float64) / d
    vn = v.astype(np.float64) / d
    nan = np.isnan(un) | np.isnan(vn)
    u0 = np.where(nan, 0.0, un)
    v0 = np.where(nan, 0.0, vn)
    rad = np.sqrt(u0 * u0 + v0 * v0)
    t = np.arctan2(-v0, -u0)
    if angle_ulps:
        t = t + angle_ulps * np.abs(np.spacing(t))
    a = t / np.pi
    fk = (a + 1) / 2 * 54 + 1
    k0 = np.clip(np.floor(fk), 1, 55).astype(np.int64)     # the clip only acts on a moved angle
    k1 = np.where(k0 + 1 == 56, 1, k0 + 1)
    f = fk - k0
    wheel = color_wheel()
    col0 = wheel[k0 - 1] / 255
    col1 = wheel[k1 - 1] / 255
    col = (1 - f)[..., None] * col0 + f[..., None] * col1
    inside = (rad <= 1)[..., None]
    col = np.where(inside, 1 - rad[..., None] * (1 - col), col * 0.75)
    pre = 255 * col * (1 - nan)[..., None]
    img = np.floor(pre)
    img[unknown] = 0
    return img.astype(np.uint8), {"maxrad": maxrad, "has_nan": has_nan, "u": un, "v": vn, "pre_floor": pre, "unknown": unknown}


def to_u8(x):
    """cv2.imwrite's convertTo(CV_8U) of a float array: round half to even, saturate to [0, 255], 0 where the rounded value is NaN or
    outside the int32 range (x86 cvtsd2si / cvtps2dq return INT_MIN there)."""
    r = np.rint(np.asarray(x, np.float64))
    bad = ~((r >= -2147483648.0) & (r <= 2147483647.0))
    return np.where(bad, 0, np.clip(np.nan_to_num(r), 0, 255)).astype(np.uint8)


def green(mask):
    """0.3 (1 - (mask > 0)) [0, 255, 0] in float64 [H, W, 3]."""
    inv = (1 - (mask > 0)[..., None]) * np.array([0, 255, 0])
    return 0.3 * inv


def composite_float(color_i, color_j, img_ij, img_ji, mask_ij, mask_ji):
    """The float64 [2H, 4W, 3] image the reference hands to cv2.imwrite (array channel order)."""
    ci, cj = color_i.astype(f32) * f32(255), color_j.astype(f32) * f32(255)
    top = np.hstack([ci, cj, img_ij.astype(f32), img_ji.astype(f32)]).astype(np.float64)
    bottom = np.hstack([(f32(0.7) * ci).astype(np.float64) + green(mask_ij), (f32(0.7) * cj).astype(np.float64) + green(mask_ji),
                        0.7 * img_ij.astype(np.float64) + green(mask_ij), 0.7 * img_ji.astype(np.float64) + green(mask_ji)])
    return np.vstack([top, bottom])


def composite(color_i, color_j, flow_ij, flow_ji, mask_ij, mask_ji):
    """vis_flow/frame_i_j.png as cv2.imread returns it ([2H, 4W, 3] u8, array channel order), and the two flow_image dicts."""
    img_ij, s_ij = flow_image(flow_ij)
    img_ji, s_ji = flow_image(flow_ji)
    return to_u8(composite_float(color_i, color_j, img_ij, img_ji, mask_ij, mask_ji)), (img_ij, s_ij), (img_ji, s_ji)


def warp_values(color, flow):
    """float32 [H, W, 3]: 255 colour sampled at pixel + flow, as grid_sample(bilinear, border, align_corners=False) of the reference's
    grid 2 uv / (W-1, H-1) - 1 computes it."""
    H, W = flow.shape[:2]
    img = color.astype(f32) * f32(255)

    def src(pix, fl, size):
        uv = pix.astype(f32) + fl
        g = f32(2) * uv / f32(size - 1) - f32(1)
        p = ((g + f32(1)) * f32(size) - f32(1)) / f32(2)
        return np.minimum(np.maximum(np.nan_to_num(p, nan=0.0, posinf=np.inf, neginf=-np.inf), f32(0)), f32(size - 1))
    with np.errstate(invalid="ignore", over="ignore"):
        px = src(np.arange(W)[None, :], flow[..., 0], W)
        py = src(np.arange(H)[:, None], flow[..., 1], H)
    x0, y0 = np.floor(px), np.floor(py)
    ix, iy = x0.astype(np.int64), y0.astype(np.int64)
    x1, y1 = x0 + f32(1), y0 + f32(1)
    out = np.zeros((H, W, 3), f32)
    for yy, xx, w in ((iy, ix, (x1 - px) * (y1 - py)), (iy, ix + 1, (px - x0) * (y1 - py)),
                      (iy + 1, ix, (x1 - px) * (py - y0)), (iy + 1, ix + 1, (px - x0) * (py - y0))):
        ok = (xx < W) & (yy < H)
        out += np.where(ok[..., None], img[np.minimum(yy, H - 1), np.minimum(xx, W - 1)] * w[..., None], f32(0))
    return out


def warp_torch(color, flow, device="cpu"):
    """The reference's warp_by_flow restated with torch (pixel grid by linspace, geometry.sample's grid, grid_sample on `device`)."""
    import torch
    H, W = flow.shape[:2]
    c = torch.from_numpy(np.ascontiguousarray(color.astype(f32) * f32(255))).permute(2, 0, 1)[None].to(device)
    fl = torch.from_numpy(np.ascontiguousarray(flow, f32)).permute(2, 0, 1)[None].to(device)
    ys, xs = torch.meshgrid(torch.linspace(0, H - 1, H, device=device), torch.linspace(0, W - 1, W, device=device), indexing="ij")
    uv = torch.stack((xs, ys))[None] + fl
    size = torch.tensor((W - 1, H - 1), dtype=uv.dtype, device=device).view(1, -1, 1, 1)
    grid = (2 * uv / size - 1).permute(0, 2, 3, 1)
    out = torch.nn.functional.grid_sample(c, grid, padding_mode="border", align_corners=False)
    return out[0].permute(1, 2, 0).contiguous().cpu().numpy()


def visualize_pair(color_i, color_j, flow_ij, flow_ji, mask_ij, mask_ji):
    """Every output of one pair (i, j): {"vis", "warp_ij" (colour j at p + flow_ij), "warp_ji", their float values, the stats}."""
    vis, (img_ij, s_ij), (img_ji, s_ji) = composite(color_i, color_j, flow_ij, flow_ji, mask_ij, mask_ji)
    wij, wji = warp_values(color_j, flow_ij), warp_values(color_i, flow_ji)
    return {"vis": vis, "warp_ij": to_u8(wij), "warp_ji": to_u8(wji), "warp_values_ij": wij, "warp_values_ji": wji,
            "flow_image_ij": img_ij, "flow_image_ji": img_ji, "stats_ij": s_ij, "stats_ji": s_ji}


def flow_image_margin(flow, ulps=4):
    """[H, W] bool: the pixels whose flow colour changes when atan2's result moves by up to `ulps` ulps either way.  CUDA's float64 atan2
    is within 2 ulps of the correctly rounded value, numpy's (glibc's) within 1; every other step of the colouring is IEEE arithmetic
    that the kernel repeats exactly, so outside these pixels the two agree."""
    base = flow_image(flow)[0]
    return ((flow_image(flow, -ulps)[0] != base) | (flow_image(flow, ulps)[0] != base)).any(axis=-1)


def round_margin(values, tol=WARP_TOL):
    """Pixels whose warp value lies within tol (1 + |v|) of a half-way point of the rounding to 8 bits.  [H, W] bool."""
    frac = np.abs(values - np.floor(values) - 0.5)
    return (frac <= tol * (1 + np.abs(values))).any(axis=-1)
