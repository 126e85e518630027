"""CPU float64 restatement of frame preparation (BaseDataset.__getitem__, src/utils/datasets.py:77-113) stage by stage, with the
arithmetic of nsb_frame.cu (include/nice_slam_b200.h, "frame preparation"): the oracle the kernel is checked against, itself checked
against cv2.undistort / cv2.resize / F.interpolate.  numpy rounds every elementwise operation on its own, so the only fused
multiply-add is the one written out (u = fx xd + cx, computed exactly through fractions where the rounding of 32 u can depend on it)."""
from fractions import Fraction

import numpy as np


def inv3(S):
    """cv::invert's closed form for a 3x3 float64 matrix: cofactors times 1/det."""
    S = np.asarray(S, dtype=np.float64).reshape(3, 3)
    det = S[0, 0] * (S[1, 1] * S[2, 2] - S[1, 2] * S[2, 1]) - S[0, 1] * (S[1, 0] * S[2, 2] - S[1, 2] * S[2, 0]) + \
        S[0, 2] * (S[1, 0] * S[2, 1] - S[1, 1] * S[2, 0])
    d = 1.0 / det
    return np.array([(S[1, 1] * S[2, 2] - S[1, 2] * S[2, 1]) * d, (S[0, 2] * S[2, 1] - S[0, 1] * S[2, 2]) * d,
                     (S[0, 1] * S[1, 2] - S[0, 2] * S[1, 1]) * d, (S[1, 2] * S[2, 0] - S[1, 0] * S[2, 2]) * d,
                     (S[0, 0] * S[2, 2] - S[0, 2] * S[2, 0]) * d, (S[0, 2] * S[1, 0] - S[0, 0] * S[1, 2]) * d,
                     (S[1, 0] * S[2, 1] - S[1, 1] * S[2, 0]) * d, (S[0, 1] * S[2, 0] - S[0, 0] * S[2, 1]) * d,
                     (S[0, 0] * S[1, 1] - S[0, 1] * S[1, 0]) * d])


def _fma_near_ties(u32, f, d, c):
    """32 * fma(f, d, c) where 32 (f d + c) lies within 1e-6 of a rounding tie (elsewhere the fused rounding cannot move rint)."""
    t = u32 - np.floor(u32)
    near = np.abs(t - 0.5) < 1e-6
    for k in zip(*np.nonzero(near)):
        u32[k] = float(Fraction(float(f)) * Fraction(float(d[k])) + Fraction(float(c))) * 32.0
    return u32


def undistort_map(H, W, fx, fy, cx, cy, dist):
    """Fixed-point source coordinates (iu, iv) int64 [H,W] (1/32 pixel) of cv2.undistort's map."""
    k1, k2, p1, p2, k3 = (float(v) for v in dist)
    iu = np.empty((H, W), np.int64)
    iv = np.empty((H, W), np.int64)
    s0 = min(max(1, 4096 // max(W, 1)), H)
    chunks = W // 8
    s = np.arange(8, dtype=np.float64)
    for row in range(H):
        y0 = row - row % s0
        ir = inv3([[fx, 0.0, cx], [0.0, fy, cy - float(y0)], [0.0, 0.0, 1.0]])
        i = float(row - y0)
        bx, by, bw = i * ir[1] + ir[2], i * ir[4] + ir[5], i * ir[7] + ir[8]
        X, Y, Wt = np.empty(W), np.empty(W), np.empty(W)
        for c in range(chunks):
            X[8 * c:8 * c + 8], Y[8 * c:8 * c + 8], Wt[8 * c:8 * c + 8] = bx + ir[0] * s, by + ir[3] * s, bw + ir[6] * s
            bx, by, bw = bx + 8.0 * ir[0], by + 8.0 * ir[3], bw + 8.0 * ir[6]
        for j in range(8 * chunks, W):
            X[j], Y[j], Wt[j] = bx, by, bw
            bx, by, bw = bx + ir[0], by + ir[3], bw + ir[6]
        w = 1.0 / Wt
        x, y = X * w, Y * w
        x2, y2 = x * x, y * y
        r2 = x2 + y2
        xy2 = 2.0 * x * y
        kr = 1.0 + ((k3 * r2 + k2) * r2 + k1) * r2
        xd = x * kr + p1 * xy2 + p2 * (r2 + 2.0 * x2)
        yd = y * kr + p1 * (r2 + 2.0 * y2) + p2 * xy2
        with np.errstate(invalid="ignore", over="ignore"):
            u32 = _fma_near_ties((fx * xd + cx) * 32.0, fx, xd, cx)
            v32 = _fma_near_ties((fy * yd + cy) * 32.0, fy, yd, cy)
        for src, dst in ((u32, iu), (v32, iv)):
            ok = (src >= -2147483648.0) & (src < 2147483647.5)
            dst[row] = np.where(ok, np.rint(np.where(ok, src, 0.0)), -2147483648).astype(np.int64)
    return iu, iv


def undistort(img, fx, fy, cx, cy, dist):
    """cv2.undistort(img u8 [H,W,3], K, dist) with BORDER_CONSTANT 0."""
    H, W = img.shape[:2]
    iu, iv = undistort_map(H, W, fx, fy, cx, cy, dist)
    sx = ((iu >> 5) + 32768) % 65536 - 32768                 # the CV_16SC2 map stores the cell as shorts
    sy = ((iv >> 5) + 32768) % 65536 - 32768
    a, b = iu & 31, iv & 31
    acc = np.zeros((H, W, 3), np.int64)
    for dy, dx, wt in ((0, 0, (32 - a) * (32 - b)), (0, 1, a * (32 - b)), (1, 0, (32 - a) * b), (1, 1, a * b)):
        X, Y = sx + dx, sy + dy
        inb = (X >= 0) & (X < W) & (Y >= 0) & (Y < H)
        v = img[np.clip(Y, 0, H - 1), np.clip(X, 0, W - 1)].astype(np.int64)
        acc += np.where(inb[..., None], v * (32 * wt)[..., None], 0)
    return np.clip((acc + (1 << 14)) >> 15, 0, 255).astype(np.uint8)


def to_rgb01(img):
    """cv2.cvtColor(BGR2RGB) / 255."""
    return img[..., ::-1].astype(np.float64) / 255.0


def _cv_coeffs(n_dst, scale):
    f = (np.arange(n_dst, dtype=np.float64) + 0.5) * scale - 0.5
    s = np.floor(f)
    return s.astype(np.int64), f - s


def cv_resize_linear(img, H, W):
    """cv2.resize(img f64 [Hs,Ws,C], (W, H)) INTER_LINEAR."""
    Hs, Ws = img.shape[:2]
    if (Hs, Ws) == (H, W):
        return img.copy()
    sx, fx = _cv_coeffs(W, 1.0 / (W / Ws))
    copy = sx + 1 >= Ws
    fx = np.where((sx < 0) | (sx >= Ws - 1), 0.0, fx)
    sx = np.clip(sx, 0, Ws - 1)
    a0, a1 = (1.0 - fx)[:, None], fx[:, None]
    sx1 = np.minimum(sx + 1, Ws - 1)
    h = np.where(copy[:, None], img[:, sx] * 1.0, img[:, sx] * a0 + img[:, sx1] * a1)          # [Hs, W, C]
    sy, fy = _cv_coeffs(H, 1.0 / (H / Hs))
    b0, b1 = (1.0 - fy)[:, None, None], fy[:, None, None]
    return h[np.clip(sy, 0, Hs - 1)] * b0 + h[np.clip(sy + 1, 0, Hs - 1)] * b1


def _torch_linear(n_out, n_in):
    if n_out == n_in:
        i = np.arange(n_out)
        return i, i, np.ones(n_out), np.zeros(n_out)
    ratio = float(n_in - 1) / float(n_out - 1) if n_out > 1 else 0.0
    real = ratio * np.arange(n_out, dtype=np.float64)
    i0 = np.minimum(np.floor(real.astype(np.float32)).astype(np.int64), n_in - 1)
    lam = np.clip(real - i0, 0.0, 1.0)
    i1 = i0 + (i0 < n_in - 1)
    return i0, i1, 1.0 - lam, lam


def interp_bilinear_ac(img, H, W):
    """F.interpolate(img.permute(2,0,1)[None], (H, W), mode='bilinear', align_corners=True) on CPU float64, back to [H,W,C]."""
    Hs, Ws = img.shape[:2]
    h0, h1, hl0, hl1 = _torch_linear(H, Hs)
    w0, w1, wl0, wl1 = _torch_linear(W, Ws)
    w00, w01 = (hl0[:, None] * wl0[None])[..., None], (hl0[:, None] * wl1[None])[..., None]
    w10, w11 = (hl1[:, None] * wl0[None])[..., None], (hl1[:, None] * wl1[None])[..., None]
    return img[h0][:, w0] * w00 + img[h0][:, w1] * w01 + img[h1][:, w0] * w10 + img[h1][:, w1] * w11


def _torch_nearest(n_out, n_in):
    i = np.arange(n_out)
    if n_out == n_in:
        return i
    if n_out == 2 * n_in:
        return i >> 1
    scale = np.float32(n_in) / np.float32(n_out)
    return np.minimum(np.floor(i.astype(np.float32) * scale).astype(np.int64), n_in - 1)


def interp_nearest(depth, H, W):
    """F.interpolate(depth[None, None], (H, W), mode='nearest')[0, 0]."""
    return depth[_torch_nearest(H, depth.shape[0])][:, _torch_nearest(W, depth.shape[1])]


def prepare(color_bgr, depth_raw, cam, scale=1.0):
    """The whole chain: (colour f64 [H,W,3], depth f32 [H,W]) from the decoded bytes, for cam = cfg['cam'] (distortion, crop_size,
    crop_edge, png_depth_scale)."""
    col = color_bgr
    if cam.get("distortion") is not None:
        col = undistort(col, cam["fx"], cam["fy"], cam["cx"], cam["cy"], cam["distortion"])
    col = to_rgb01(col)
    depth = (depth_raw.astype(np.float32) / np.float32(cam["png_depth_scale"])) * np.float32(scale)
    H, W = depth.shape
    col = cv_resize_linear(col, H, W)
    if cam.get("crop_size") is not None:
        ch, cw = cam["crop_size"]
        col = interp_bilinear_ac(col, ch, cw)
        depth = interp_nearest(depth, ch, cw)
    e = int(cam.get("crop_edge", 0))
    if e > 0:
        col, depth = col[e:-e, e:-e], depth[e:-e, e:-e]
    return np.ascontiguousarray(col), np.ascontiguousarray(depth)
