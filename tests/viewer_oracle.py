"""Vectorised numpy checker of the headless viewer (csrc/viewer.cu) -- TEST INFRASTRUCTURE ONLY.

It restates PointsColorUpdater::update (points_color_updater.cpp:37-61) and the overlay's rules on top of the CPU oracle's
projection and estimate_camera_fov (oracle/oracle.py): the transform in Eigen's operation order in float64, the FoV test
on the normalised z, truncation toward zero with x86's out-of-range result, the bounds test, and the blend in float32
with one rounding per operation (numpy never fuses a multiply and an add).  The Turbo table comes from OpenCV, not from
the library."""
import numpy as np

INT_MIN = -(2**31)


def turbo_table():
    """cv2.COLORMAP_TURBO as (256, 3) uint8 RGB."""
    import cv2

    return cv2.applyColorMap(np.arange(256, dtype=np.uint8).reshape(-1, 1), cv2.COLORMAP_TURBO).reshape(256, 3)[:, ::-1].copy()


def viewer_cos_fov(O, cam, W, H):
    """min_nz of points_color_updater.cpp:27: the viewer's threshold, half a degree looser than the cost's."""
    return float(np.cos(O.estimate_camera_fov(cam, W, H) + 0.5 * np.pi / 180.0))


def cost_cos_fov(O, cam, W, H):
    return float(np.cos(O.estimate_camera_fov(cam, W, H)))


def _cast_int_x86(v):
    ok = (v > -2147483649.0) & (v < 2147483648.0)
    return np.where(ok, np.trunc(np.where(ok, v, 0.0)), INT_MIN).astype(np.int64)


def classify(O, cam, W, H, cos_fov, T, points):
    """-> (pixel iy * W + ix of every point, -1 where the reference skips it; squared range in Eigen's order)."""
    T = np.asarray(T, dtype=np.float64)
    p = np.asarray(points, dtype=np.float64)
    x, y, z = p[:, 0], p[:, 1], p[:, 2]
    with np.errstate(all="ignore"):
        pc = [((T[r, 0] * x + T[r, 1] * y) + T[r, 2] * z) + T[r, 3] for r in range(3)]
        n2 = (pc[0] * pc[0] + pc[1] * pc[1]) + pc[2] * pc[2]
        nz = np.where(n2 > 0.0, pc[2] / np.sqrt(n2), pc[2])
        in_fov = ~(nz < cos_fov)
        uv = O.project(cam, np.stack(pc, axis=1)) if len(p) else np.zeros((0, 2))
    ix, iy = _cast_int_x86(uv[:, 0]), _cast_int_x86(uv[:, 1])
    ok = in_fov & (ix >= 0) & (iy >= 0) & (ix < W) & (iy < H)
    return np.where(ok, iy * W + ix, -1), n2


def turbo_index(intensities):
    with np.errstate(all="ignore"):
        v = np.asarray(intensities, dtype=np.float64).astype(np.float32).astype(np.float64) * 255.0
    idx = np.zeros(v.shape, dtype=np.int64)  # negative, zero and NaN
    pos = v > 0.0
    idx[pos] = np.trunc(np.minimum(v[pos], 255.0)).astype(np.int64)
    return idx


def blend(gray_u8, intensities, w):
    """gray * w + turbo * (1 - w), alpha w + (1 - w): (N, 4) float32, one float32 rounding per operation."""
    w = np.float32(w)
    omw = np.float32(1.0 - float(w))  # 1 - w in double, then rounded
    f255 = np.float32(255.0)
    gray = (np.asarray(gray_u8).astype(np.float32) / f255) * w
    turbo = (turbo_table()[turbo_index(intensities)].astype(np.float32) / f255) * omw
    out = np.empty((len(gray), 4), dtype=np.float32)
    out[:, :3] = gray[:, None] + turbo
    out[:, 3] = w + omw
    return out


def colorize(O, cam, image, T, points, intensities, w):
    """PointsColorUpdater::update -> (N, 4) float32."""
    H, W = image.shape
    pix, _ = classify(O, cam, W, H, viewer_cos_fov(O, cam, W, H), T, points)
    out = np.zeros((len(pix), 4), dtype=np.float32)
    m = pix >= 0
    out[m] = blend(image.reshape(-1)[pix[m]], np.asarray(intensities)[m], w)
    return out


def overlay(O, cam, image, T, points, intensities, radius, w):
    """-> (BGR uint8 (H, W, 3), winner index int32 (H, W)): per pixel, among the points whose square of `radius` covers it,
    the smallest squared range, of equal ones the largest index."""
    H, W = image.shape
    pix, n2 = classify(O, cam, W, H, cost_cos_fov(O, cam, W, H), T, points)
    idx = np.nonzero(pix >= 0)[0]
    iy, ix = pix[idx] // W, pix[idx] % W
    key = n2[idx].view(np.uint64)  # non-negative doubles order like their bit patterns
    zmin = np.full(H * W, np.float64(np.finfo(np.float64).max).view(np.uint64), dtype=np.uint64)
    index = np.full(H * W, -1, dtype=np.int64)
    offsets = [(dy, dx) for dy in range(-radius, radius + 1) for dx in range(-radius, radius + 1)]
    cover = []
    for dy, dx in offsets:
        yy, xx = iy + dy, ix + dx
        m = (yy >= 0) & (yy < H) & (xx >= 0) & (xx < W)
        cover.append((yy[m] * W + xx[m], m))
        np.minimum.at(zmin, cover[-1][0], key[m])
    for p, m in cover:
        won = key[m] == zmin[p]
        np.maximum.at(index, p[won], idx[m][won])
    index = index.reshape(H, W)
    bgr = np.repeat(image[:, :, None], 3, axis=2).copy()
    hit = index >= 0
    c = blend(image[hit], np.asarray(intensities)[index[hit]], w)
    bgr[hit] = np.clip(np.rint(c[:, 2::-1] * np.float32(255.0)), 0, 255).astype(np.uint8)
    return bgr, index.astype(np.int32)


def overlay_serial(O, cam, image, T, points, intensities, radius, w):
    """The index map of overlay() by the reference's serial rule (generate_lidar_image.cpp:31-37 per covered pixel): a
    point replaces the pixel's winner unless the stored squared range is strictly smaller.  Small inputs only."""
    H, W = image.shape
    pix, n2 = classify(O, cam, W, H, cost_cos_fov(O, cam, W, H), T, points)
    best = np.full((H, W), np.finfo(np.float64).max)
    index = np.full((H, W), -1, dtype=np.int32)
    for i in np.nonzero(pix >= 0)[0]:
        y, x = divmod(int(pix[i]), W)
        for yy in range(max(y - radius, 0), min(y + radius, H - 1) + 1):
            for xx in range(max(x - radius, 0), min(x + radius, W - 1) + 1):
                if best[yy, xx] < n2[i]:
                    continue
                best[yy, xx], index[yy, xx] = n2[i], i
    return index
