"""Writes tests/golden/flow_register_golden.npz from the reference's own optical_flow_homography (imported unchanged):

    python tests/golden/make_flow_register_golden.py <reference checkout>

Each case is a pair of seeded BGR frames written as color_flow PNGs.  SURF is absent from stock cv2, so the reference's
detectAndDescribe is replaced by the same function on cv2.SIFT_create; the model is the deterministic stub below (fractional flows that
depend on both images).  Per case the fixture holds the frames, the reference's H_BA and img2_registered (getimage), the model's flow,
the flows before and after resize_flow (infer, resize_flow) and the bytes save_raw_float32_image writes."""
import os
import sys
import tempfile

import cv2
import numpy as np
import torch


def stub_model(img1, img2, iters=20, test_mode=True):
    """(flow_low, flow_up) of a [1, 3, H, W] pair: smooth fractional flows plus a term of both images."""
    _, _, H, W = img1.shape
    yy, xx = torch.meshgrid(torch.arange(H, dtype=torch.float32), torch.arange(W, dtype=torch.float32), indexing="ij")
    d = (img1 - img2).mean(1)[0] / 255
    u = 1.7 * torch.sin(xx * 0.05) + 0.25 * d + 0.125
    v = -1.3 * torch.cos(yy * 0.07) - 0.25 * d
    up = torch.stack([u, v])[None]
    return up / 8, up


def texture(rng, H, W):
    """A blurred random BGR image with structure at several scales (SIFT finds keypoints on it)."""
    img = np.zeros((H, W, 3), np.float64)
    for s in (2, 5, 13):
        n = rng.random((H // s + 2, W // s + 2, 3))
        img += cv2.resize(n, (W, H), interpolation=cv2.INTER_CUBIC) * s
    img = (img - img.min()) / (img.max() - img.min()) * 255
    return np.clip(img, 0, 255).astype(np.uint8)


def cases():
    rng = np.random.default_rng(20261019)
    H1 = np.array([[1.02, 0.03, -4.5], [-0.02, 0.99, 3.25], [1.5e-4, -1e-4, 1.0]])
    H2 = np.array([[0.97, -0.05, 6.0], [0.04, 1.03, -2.5], [-3e-4, 2e-4, 1.0]])
    out = []
    a = texture(rng, 72, 128)
    out.append(("perspective", a, cv2.warpPerspective(a, H1, (128, 72), borderMode=cv2.BORDER_REFLECT), (48, 28)))
    b = texture(rng, 61, 97)
    out.append(("odd_size", b, cv2.warpPerspective(b, H2, (97, 61), borderMode=cv2.BORDER_REFLECT), (41, 23)))
    c = texture(rng, 48, 80)
    out.append(("same_size", c, np.roll(c, (2, -3), (0, 1)), (80, 48)))
    flat = np.full((40, 64, 3), 128, np.uint8)
    out.append(("no_keypoints", flat, flat.copy(), (24, 16)))
    out.append(("unrelated", texture(rng, 64, 96), texture(rng, 64, 96), (40, 24)))
    out.append(("upscale", texture(rng, 32, 48), texture(rng, 32, 48), (72, 40)))
    return out


def main(ref):
    sys.path.insert(0, ref)
    import optical_flow_homography as ofh
    from utils.image_io import save_raw_float32_image

    def sift_describe(image):
        kps, features = cv2.SIFT_create().detectAndCompute(image, None)
        return np.float32([kp.pt for kp in kps]), features
    ofh.detectAndDescribe = sift_describe

    class Args:
        homography = True
        model = "raft"

    arrays = {}
    names = []
    with tempfile.TemporaryDirectory() as tmp:
        for name, f1, f2, size in cases():
            p1, p2, raw = (os.path.join(tmp, n) for n in ("frame1.png", "frame2.png", "flow.raw"))
            cv2.imwrite(p1, f1)
            cv2.imwrite(p2, f2)
            img1, _, reg, H_BA = ofh.getimage(p1, p2)
            with torch.no_grad():
                _, up = stub_model(img1[None], reg[None])
            flow = ofh.infer(Args, stub_model, torch.device("cpu"), p1, p2)
            resized = ofh.resize_flow(flow, size)
            save_raw_float32_image(raw, resized)
            with open(raw, "rb") as f:
                raw_bytes = np.frombuffer(f.read(), np.uint8)
            arrays.update({f"{name}/frame1": cv2.imread(p1), f"{name}/frame2": cv2.imread(p2), f"{name}/H_BA": H_BA,
                           f"{name}/registered": reg.permute(1, 2, 0).numpy().astype(np.uint8),
                           f"{name}/model_flow": up[0].permute(1, 2, 0).numpy(), f"{name}/flow": flow, f"{name}/resized": resized,
                           f"{name}/raw": raw_bytes, f"{name}/size": np.array(size)})
            names.append(name)
    arrays["cases"] = np.array(names)
    arrays["cv2_version"] = np.array(cv2.__version__)
    out = os.path.join(os.path.dirname(os.path.abspath(__file__)), "flow_register_golden.npz")
    np.savez_compressed(out, **arrays)
    print(f"wrote {out}: {', '.join(names)}")


if __name__ == "__main__":
    main(sys.argv[1] if len(sys.argv) > 1 else "/path/to/robust_cvd")
