"""numpy restatement of the per-frame post-processing of the reference's dynamic_mask_generation (dynamic_mask_generation.py:143-182):
the union of the dynamic instances, cv2.dilate(mask, np.ones((d, d), np.uint8)), cv2.bitwise_not and the --save_anno image.  The
dilation is written from its definition (a window of d rows and columns starting d // 2 before the pixel, clipped to the image, d = 0
meaning 3), by prefix sums, so it shares nothing with the kernels' running scans.  `reference_frame` replays the reference's own
numpy / cv2 calls for one frame."""
import numpy as np

DYNAMIC = frozenset(list(range(0, 8)) + list(range(13, 23)))


def window_any(m, d, axis):
    """Whether any element of the boolean array m is set in the window [i - d // 2, i - d // 2 + d - 1] along `axis`, clipped."""
    a = d // 2
    n = m.shape[axis]
    c = np.concatenate([np.zeros_like(np.take(m, [0], axis=axis), np.int64), np.cumsum(m, axis=axis, dtype=np.int64)], axis=axis)
    lo = np.clip(np.arange(n) - a, 0, n)
    hi = np.clip(np.arange(n) - a + d, 0, n)
    return (np.take(c, hi, axis=axis) - np.take(c, lo, axis=axis)) > 0


def dilate(mask, d):
    """cv2.dilate(mask, np.ones((d, d), np.uint8), iterations=1) of a 0 / 255 u8 mask."""
    if d < 0:
        raise ValueError("negative dilation")
    d = 3 if d == 0 else d
    m = mask != 0
    return (window_any(window_any(m, d, 0), d, 1) * 255).astype(np.uint8)


def union(instances, shape):
    """u8 [h, w]: 255 where any of the boolean instances [K, h, w] is set."""
    out = np.zeros(shape, np.uint8)
    if len(instances):
        out[np.any(np.asarray(instances) != 0, axis=0)] = 255
    return out


def frame_outputs(img_bgr, classes, masks, d, save_anno=True):
    """(mask written as <base>.png, the anonymised image as stored by cv2.imwrite in R, G, B order or None) for one frame."""
    sel = [k for k, c in enumerate(classes) if int(c) in DYNAMIC]
    u = union(np.asarray(masks)[sel] if sel else np.zeros((0,) + img_bgr.shape[:2], bool), img_bgr.shape[:2])
    anon = None
    if save_anno:
        anon = img_bgr[:, :, ::-1].copy()
        anon[u != 0] = 255
    return 255 - dilate(u, d), anon


def reference_frame(img_bgr, classes, masks, d, save_anno=True):
    """The reference's own per-frame calls (boolean-index writes, cv2.dilate, cv2.bitwise_not), with the anonymised image returned as
    B, G, R (cv2.imwrite's input)."""
    import cv2
    mask_img = np.transpose(np.copy(img_bgr), (2, 0, 1)).astype(np.uint8)
    mask = np.zeros(img_bgr.shape[:2]).astype(np.uint8)
    for idx, c in enumerate(classes):
        if int(c) in DYNAMIC:
            m = np.asarray(masks[idx])
            mask[m] = 255
            if save_anno:
                for ch in range(3):
                    mask_img[ch][m] = 255
    mask = cv2.dilate(mask, kernel=np.ones((d, d), dtype=np.uint8), iterations=1)
    return cv2.bitwise_not(mask), (np.transpose(mask_img, (1, 2, 0)) if save_anno else None)
