"""Pins the bag checker (tests/cpp/bag_oracle.c) and the host restatements of `preprocess` to the reference's OWN code:
extract_raw_points, TimeKeeper::process and the static integrator, compiled where they lie (oracle/bag_ref.mk) and
recorded on the scans below in tests/golden/reference_bag_outputs.json (tests/golden/make_reference_bag_outputs.py).
Checked: extracted fields bit for bit (z read with x's datatype, every intensity datatype, times) and the scans the
reference refuses; TimeKeeper skip decisions; the integrated rows as a multiset, and the checker's order equal to
first-write order."""
import json
import math
import os

import numpy as np
import pytest

import bag_oracle as BO
import bag_writer as BW
from direct_visual_lidar_calibration_b200 import _lib as VL
from direct_visual_lidar_calibration_b200 import preprocess_bag as PB

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "reference_bag_outputs.json")
DT = {2: "u1", 3: "<i2", 4: "<u2", 6: "<u4", 7: "<f4", 8: "<f8"}


def _layout_scan(rng, n, xt, it, tt=None, z_type=None, channel="intensity", extra=()):
    """-> (data, width, height, point_step, fields [(name, offset, datatype)], channel); unaligned offsets, padded step."""
    xs = np.dtype(DT[xt]).itemsize
    off = {"x": 1, "y": 1 + xs, "z": 1 + 2 * xs}
    pos = 1 + 3 * xs + 1
    off["intensity"] = pos
    pos += np.dtype(DT[it]).itemsize
    if tt is not None:
        off["time"] = pos
        pos += np.dtype(DT[tt]).itemsize
    step = pos + 5
    buf = np.zeros((n, step), np.uint8)
    xyz = rng.normal(0.0, 20.0, (n, 3))

    def put(name, vals, t):
        a = np.asarray(vals).astype(DT[t])
        buf[:, off[name]:off[name] + a.itemsize] = a.view(np.uint8).reshape(n, a.itemsize)

    for k, c in enumerate("xyz"):
        put(c, xyz[:, k], xt)
    top = {2: 255, 3: 3000, 4: 65535, 6: 2**32 - 1}.get(it, 1e5)
    put("intensity", rng.uniform(0, top, n), it)
    if tt is not None:
        base = {6: 0, 7: 0.0, 8: 1.7e9}[tt]
        put("time", base + np.sort(rng.uniform(0, 0.1 if tt != 6 else 1e8, n)), tt)
    fields = [("x", off["x"], xt), ("y", off["y"], xt), ("z", off["z"], z_type or xt), ("intensity", off["intensity"], it)]
    if tt is not None:
        fields.append(("time", off["time"], tt))
    return buf.tobytes(), n, 1, step, fields + list(extra), channel


def extraction_cases():
    rng = np.random.default_rng(11)
    cases = {}
    for xt in (7, 8):
        for it in (2, 4, 6, 7, 8):
            cases[f"x{xt}_i{it}"] = _layout_scan(rng, 64, xt, it, tt=[6, 7, 8][it % 3])
    cases["z_declared_f64_read_as_f32"] = _layout_scan(rng, 32, 7, 7, z_type=8)
    cases["z_declared_f32_read_as_f64"] = _layout_scan(rng, 32, 8, 7, z_type=7)
    data, w, h, step, fields, ch = _layout_scan(rng, 16, 7, 7)
    cases["missing_y"] = (data, w, h, step, [f for f in fields if f[0] != "y"], ch)
    cases["x_y_types_differ"] = (data, w, h, step, [fields[0], (fields[1][0], fields[1][1], 8)] + fields[2:], ch)
    cases["x_int32"] = (data, w, h, step, [(f[0], f[1], 5) if f[0] in "xy" else f for f in fields], ch)
    cases["intensity_int16"] = _layout_scan(rng, 16, 7, 3)
    cases["time_uint16"] = (data, w, h, step, fields + [("t", 0, 4)], ch)
    cases["channel_is_x"] = (data, w, h, step, fields, "x")
    cases["no_points_bad_intensity_type"] = (b"", 0, 1, step, [(f[0], f[1], 3) if f[0] == "intensity" else f for f in fields], ch)
    return cases


def time_keeper_cases():
    rng = np.random.default_rng(12)
    rel = [np.sort(rng.uniform(0, 0.1, 50)) for _ in range(6)]
    return {
        "no_times": [(10.0, 5, []), (10.1, 5, []), (10.05, 5, []), (10.2, 5, []), (10.2, 0, [])],
        "relative": [(5.0, 50, rel[0]), (4.0, 50, rel[1]), (6.0, 50, rel[2])],
        "absolute_near": [(100.0, 3, [100.5, 100.55, 100.6]), (100.9, 3, [100.4, 100.45, 100.5]), (101.0, 3, [100.7, 100.8, 100.9])],
        "absolute_far_offset": [(1000.0, 2, [10.0, 10.1]), (5.0, 2, [10.2, 10.3]), (2000.0, 2, [10.1, 10.15])],
        "nanoseconds": [(2.0e7, 2, [2.0e16, 2.0e16 + 5e7]), (2.0e7, 2, [2.0e16 - 1e9, 2.0e16])],
        "negative": [(50.0, 3, [-0.05, 0.0, 0.02]), (50.0, 3, [0.0, -0.1, 0.02]), (49.0, 3, [-0.01, 0.0, 0.01])],
        "mixed": [(3.0, 0, []), (3.1, 2, [3.1, 3.2]), (2.0, 2, []), (3.5, 2, [0.0, 0.05])],
    }


def integration_cases():
    rng = np.random.default_rng(13)
    cases = {}
    frames = []
    base = rng.uniform(-5.0, 5.0, (60, 3))
    for k in range(5):  # the same voxels rewritten by every frame
        frames.append((base + rng.normal(0.0, 0.004, base.shape), rng.uniform(0, 255, 60)))
    cases["rewrites"] = (frames, 0.05, 1.0)
    d = rng.normal(size=(200, 3))
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    edge = np.concatenate([d, d * np.nextafter(1.0, 2.0), d * np.nextafter(1.0, 0.0), [[1.5, 0, 0], [np.nextafter(1.5, 0), 0, 0]]])
    cases["min_distance_edges"] = ([(edge, np.arange(edge.shape[0], dtype=np.float64))], 0.001, 1.0)
    k = rng.integers(-300, 300, (300, 3)) * 0.05
    vox = np.concatenate([k, np.nextafter(k, np.inf), np.nextafter(k, -np.inf)])
    cases["voxel_edges"] = ([(vox[:450], rng.uniform(0, 1, 450)), (vox[450:], rng.uniform(0, 1, vox.shape[0] - 450))], 0.05, 1.0)
    far = rng.uniform(-50.0, 50.0, (200, 3))
    far[:100, 0] += 5.0e6
    far[100:, 2] -= 5.0e7
    cases["int_min"] = ([(far, rng.uniform(0, 1, 200))], 0.002, 1.0)
    cases["default_resolution"] = ([(rng.uniform(-3, 3, (500, 3)), rng.uniform(0, 100, 500)) for _ in range(3)], 0.002, 1.0)
    return cases


def reference_outputs(R):
    """What the reference's compiled code returns on the cases above (float64 arrays as hex of their bytes)."""
    hx = lambda a: np.ascontiguousarray(a, np.float64).tobytes().hex()  # noqa: E731
    out = {"extract": {}, "time_keeper": {}, "integrate": {}}
    for name, (data, w, h, step, fields, ch) in extraction_cases().items():
        r = R.extract(data, w, h, step, fields, ch)
        out["extract"][name] = None if r is None else {"points": hx(r["points"]), "intensities": hx(r["intensities"]), "times": hx(r["times"])}
    for name, frames in time_keeper_cases().items():
        out["time_keeper"][name] = R.time_keeper(frames)
    for name, (frames, res, md) in integration_cases().items():
        out["integrate"][name] = hx(R.integrate(frames, res, md))
    return out


def _golden():
    with open(GOLDEN) as f:
        return json.load(f)


def _f64(h):
    return np.frombuffer(bytes.fromhex(h), np.float64)


@pytest.mark.parametrize("name", sorted(extraction_cases()))
def test_extraction_matches_the_reference(name):
    data, w, h, step, fields, ch = extraction_cases()[name]
    ref = _golden()["extract"][name]
    msg = {"fields": [(n, o, t, 1) for n, o, t in fields], "width": w, "height": h, "point_step": step, "data": data}
    if ref is None:
        with pytest.raises(PB.Unconvertible):
            PB.scan_layout(msg, ch)
        return
    n, (xo, yo, zo), xt, tf, (io, it) = PB.scan_layout(msg, ch)
    pts = _f64(ref["points"]).reshape(-1, 4)
    assert n == pts.shape[0]
    if n == 0:
        return
    desc = VL.ScanDesc(byte_offset=0, n_points=n, point_step=step, x_offset=xo, y_offset=yo, z_offset=zo, xyz_type=xt, intensity_offset=io, intensity_type=it)
    got = BO.extract_scan(np.frombuffer(data, np.uint8), desc)
    assert got[:, :3].tobytes() == pts[:, :3].tobytes()
    assert got[:, 3].tobytes() == _f64(ref["intensities"]).tobytes()
    times = _f64(ref["times"])
    summary = PB.point_times(msg, n, tf)
    assert (summary is None) == (times.size == 0)
    if summary is not None:
        assert summary == (times[0], times[-1], times.min())


@pytest.mark.parametrize("name", sorted(time_keeper_cases()))
def test_time_keeper_matches_the_reference(name):
    tk = PB.TimeKeeper()
    got = []
    for stamp, n, times in time_keeper_cases()[name]:
        t = np.asarray(times, np.float64)
        got.append(tk.process(stamp, (t[0], t[-1], t.min()) if n > 0 and t.size else None))
    assert got == _golden()["time_keeper"][name]


def _first_write_order(frames, res, md):
    """insert_points restated with a dict: insertion order is first-write order, values are the last write."""
    d2i = lambda v: int(v) if -2147483648.0 <= v < 2147483648.0 else -2147483648  # noqa: E731
    vox = {}
    for pts, inten in frames:
        for (x, y, z), w in zip(np.asarray(pts, np.float64).tolist(), np.asarray(inten, np.float64).tolist()):
            if math.sqrt((x * x + y * y) + z * z) < md:
                continue
            vox[(d2i(math.floor(x / res)), d2i(math.floor(y / res)), d2i(math.floor(z / res)))] = (x, y, z, w)
    return np.array(list(vox.values()), np.float64).reshape(-1, 4).astype(np.float32)


@pytest.mark.parametrize("name", sorted(integration_cases()))
def test_integration_matches_the_reference(name):
    frames, res, md = integration_cases()[name]
    scans = []
    for pts, inten in frames:
        data, fields, step = BW.cloud_bytes(np.asarray(pts), np.asarray(inten), "<f8", "<f8")
        scans.append((data, {n: (o, t) for n, o, t in fields}, step, len(pts)))
    parts, descs, off = [], [], 0
    for data, f, step, n in scans:
        descs.append(VL.ScanDesc(byte_offset=off, n_points=n, point_step=step, x_offset=f["x"][0], y_offset=f["y"][0], z_offset=f["z"][0],
                                 xyz_type=f["x"][1], intensity_offset=f["intensity"][0], intensity_type=f["intensity"][1]))
        parts.append(np.frombuffer(data, np.uint8))
        off += len(data)
    got, _ = BO.bag_integrate(np.concatenate(parts), descs, res, md)
    ref = _f64(_golden()["integrate"][name]).reshape(-1, 4).astype(np.float32)  # get_points' float casts (exact here)
    key = lambda a: sorted(bytes(r) for r in np.ascontiguousarray(a))  # noqa: E731
    assert got.shape == ref.shape and key(got) == key(ref)  # the same rows as a multiset
    assert got.tobytes() == _first_write_order(frames, res, md).tobytes()  # in first-write order
