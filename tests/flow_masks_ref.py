"""CPU restatement of the flow-consistency masks (the reference's consistent_flow_masks, utils/consistency.py): numpy for the
target positions, the tests and the sse, and torch.nn.functional.grid_sample on CPU tensors for the sampling, which is what the
reference runs.  Besides the masks it returns what the GPU tests compare: the sampled arrays and the sse values of each direction.

sample_fma() is the same sampling written out in float32 with fused multiply-adds (emulated exactly in float64: a float32 product is
exact in float64 and the one rounding of the sum is followed by a rounding to float32 that is exact unless the float64 sum lies on a
float32 midpoint).  It is the formulation rcvd_flowmask.cuh computes; on x86 hosts whose torch runs the vectorised (AVX2 / AVX-512)
grid_sample kernel it equals torch's CPU result bit for bit."""
import numpy as np
import torch

f32 = np.float32


def target_positions(flow):
    """(X, Y) = pixel + flow in float64 (a float32 plus an integer is exact in float64) and the in-image test (NaN fails)."""
    H, W = flow.shape[:2]
    X = np.arange(W)[None, :] + flow[..., 0].astype(np.float64)
    Y = np.arange(H)[:, None] + flow[..., 1].astype(np.float64)
    inside = (X >= 0) & (X <= W - 1) & (Y >= 0) & (Y <= H - 1)
    return X, Y, inside


def grid(X, Y, W, H):
    """grid_sample's normalised grid: 2 X / W - 1 in float64, then rounded to float32, as the reference builds it."""
    return np.stack(((2 * X / W - 1).astype(np.float32), (2 * Y / H - 1).astype(np.float32)), axis=-1)


def sample_torch(img, g):
    """grid_sample(bilinear, border, align_corners=False) of img [H, W, C] f32 at g [H, W, 2] on CPU."""
    t = torch.from_numpy(np.ascontiguousarray(img)).permute(2, 0, 1)[None]
    out = torch.nn.functional.grid_sample(t, torch.from_numpy(np.ascontiguousarray(g))[None], mode="bilinear", padding_mode="border",
                                          align_corners=False)
    return out[0].permute(1, 2, 0).contiguous().numpy()


def _fma(a, b, c):
    return (a.astype(np.float64) * b.astype(np.float64) + c.astype(np.float64)).astype(np.float32)


def sample_fma(img, g):
    """sample_torch in float32 with fused multiply-adds: p = fma(g + 1, size / 2, -0.5) clamped to [0, size-1], weights from floor(p),
    taps summed as fma(se, w_se, fma(sw, w_sw, fma(ne, w_ne, nw * w_nw))), a tap past the last row / column reading 0."""
    H, W, C = img.shape

    def src(gc, size):
        p = _fma(gc + f32(1), np.full_like(gc, f32(size) / f32(2)), np.full_like(gc, f32(-0.5)))
        return np.minimum(np.maximum(np.nan_to_num(p, nan=0.0), f32(0)), f32(size - 1))
    px, py = src(g[..., 0], W), src(g[..., 1], H)
    xw, yn = np.floor(px), np.floor(py)
    w = px - xw; e = f32(1) - w; n = py - yn; s = f32(1) - n
    ix, iy = xw.astype(np.int64), yn.astype(np.int64)

    def tap(yy, xx):
        v = img[np.minimum(yy, H - 1), np.minimum(xx, W - 1)]
        return np.where(((xx < W) & (yy < H))[..., None], v, f32(0))

    def wt(a):
        return np.broadcast_to(a[..., None], ix.shape + (C,))
    acc = tap(iy, ix) * wt(s * e)
    acc = _fma(tap(iy, ix + 1), wt(s * w), acc)
    acc = _fma(tap(iy + 1, ix), wt(n * e), acc)
    return _fma(tap(iy + 1, ix + 1), wt(n * w), acc)


def sse(a, b):
    """d0^2 + d1^2 (+ d2^2) in float32, summed in that order (numpy's order for a last axis of 2 or 3)."""
    d = a - b
    q = d * d
    out = q[..., 0] + q[..., 1]
    return out + q[..., 2] if q.shape[-1] == 3 else out


def direction(flow_ref, flow_tgt, color_ref, color_tgt, flow_thresh_sq, color_thresh_sq, sampler=sample_torch):
    """One direction: ref -> tgt along flow_ref.  Returns the mask (bool) and the sampled arrays and sse values of both checks."""
    H, W = flow_ref.shape[:2]
    X, Y, inside = target_positions(flow_ref)
    g = grid(X, Y, W, H)
    flow_s = sampler(-flow_tgt, g)
    color_s = sampler(color_tgt, g)
    sf, sc = sse(flow_ref, flow_s), sse(color_ref, color_s)
    mask = inside & (sf < f32(flow_thresh_sq)) & (sc < f32(color_thresh_sq))
    return {"mask": mask, "flow_sample": flow_s, "color_sample": color_s, "sse_flow": sf, "sse_color": sc, "nan_pos": np.isnan(X) | np.isnan(Y)}


def thresholds(flow_thresh=1, color_thresh=1, channels=3):
    """The float32 thresholds the reference's comparisons use: flow_thresh^2 and C color_thresh^2."""
    return f32(flow_thresh ** 2), f32(channels * color_thresh ** 2)


def flow_masks(flow_ij, flow_ji, color_i, color_j, flow_thresh=1, color_thresh=1, sampler=sample_torch):
    """Both directions of a pair: ([i -> j, j -> i] direction dicts)."""
    fsq, csq = thresholds(flow_thresh, color_thresh, color_i.shape[-1])
    return [direction(flow_ij, flow_ji, color_i, color_j, fsq, csq, sampler), direction(flow_ji, flow_ij, color_j, color_i, fsq, csq, sampler)]


def torch_is_vectorised():
    """True when torch's CPU kernels run an x86 vector ISA with FMA (AVX2 / AVX-512), where sample_torch == sample_fma bit for bit."""
    try:
        return torch.backends.cpu.get_cpu_capability() in ("AVX2", "AVX512")
    except Exception:
        return False
