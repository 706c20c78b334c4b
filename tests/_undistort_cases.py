"""Cameras and point sets for the lens-undistortion tests, with the branches of the inverse maps each one reaches.

The definition being tested is ``cv2.undistortPoints`` / ``cv2.fisheye.undistortPoints`` on float32 copies of the
points with ``P=None`` (normalised output) or ``P=K`` (pixels), float32 results.  The cameras cover every coefficient
count the C ABI takes (0, 4, 5, 8 and 12 Brown-Conrady coefficients, each with and without skew) and fisheye lenses
that reach the Newton iteration's failure sentinel and its ``|theta_d| <= 1e-8`` branch; the points cover the image,
three image sizes around it, the principal point, doubles that round on the way to float32 and non-finite rows."""
from __future__ import annotations

from dataclasses import dataclass, field

import numpy as np

W, H = 1280, 960
SENTINEL = -1000000.0  # cv2.fisheye.undistortPoints' value for a point whose Newton iteration fails or flips sign


@dataclass(frozen=True)
class Cam:
    name: str
    K: np.ndarray
    d: np.ndarray
    fisheye: bool
    reaches: frozenset = field(default_factory=frozenset)  # branches (see `branches`) its points must reach


def _K(fx, fy, cx, cy, skew=0.0):
    return np.array([[fx, skew, cx], [0.0, fy, cy], [0.0, 0.0, 1.0]])


_PINHOLE = {
    # "no distortion" as the reference stores it: a zero coefficient vector (cv2 then still runs the iteration)
    "pin0": [0.0] * 5,
    "pin4": [-0.21, 0.07, 0.0012, -0.0008],
    "pin5": [-0.28, 0.09, 0.001, -0.0007, -0.012],
    "pin5_barrel": [-0.9, 0.6, 0.0, 0.0, -0.3],
    "pin8": [0.4, -0.2, 0.001, -0.0007, 0.05, 0.7, -0.1, 0.08],
    "pin12": [-0.2, 0.05, 0.001, -0.0007, 0.01, 0.1, 0.02, 0.0, 0.003, -0.001, 0.002, 0.0005],
}


def cameras() -> list[Cam]:
    out = []
    for name, d in _PINHOLE.items():
        for skew in (0.0, 2.5):
            reaches = {"nonfinite"} | ({"icdist_neg"} if name == "pin5_barrel" else set())
            out.append(Cam(name + ("_skew" if skew else ""), _K(912.7, 905.3, 651.3, 472.9, skew), np.array(d), False,
                           frozenset(reaches)))  # fmt: skip
    mild = np.array([0.02, -0.01, 0.003, -0.001])
    out += [
        Cam("fish_mild", _K(601.3, 598.9, 641.7, 478.2), mild, True, frozenset({"nonfinite"})),
        Cam("fish_wild", _K(600.0, 600.0, 640.0, 480.0), np.array([-0.5, 0.3, -0.2, 0.05]), True,
            frozenset({"nonfinite", "sentinel"})),
        Cam("fish_skew", _K(601.3, 598.9, 641.7, 478.2, 1.5), mild, True, frozenset({"nonfinite"})),
        # near cx = 640 the float32 pixel closest to cx is 6e-5 px away (1e-7 f), so only a principal point near 0
        # puts pixels inside theta_d in (0, 1e-8]
        Cam("fish_c0", _K(600.0, 600.0, 0.25, 0.25), mild, True, frozenset({"nonfinite", "theta_tiny"})),
    ]  # fmt: skip
    return out


NONFINITE = np.array([[np.nan, 100.0], [100.0, np.nan], [np.nan, np.nan], [np.inf, 100.0], [-np.inf, 100.0],
                      [100.0, np.inf], [100.0, -np.inf], [np.inf, -np.inf], [np.nan, -np.inf]])  # fmt: skip


def point_sets(cam: Cam, seed: int = 0) -> dict[str, np.ndarray]:
    """Named (n, 2) float64 point sets for `cam`."""
    rng = np.random.default_rng(seed)
    cx, cy = cam.K[0, 2], cam.K[1, 2]
    gx, gy = np.meshgrid(np.linspace(0.0, W, 41), np.linspace(0.0, H, 31))
    f32 = np.float32
    # the principal point and its float32 neighbours (one and two steps away in each direction)
    near = []
    for a in (-2, -1, 0, 1, 2):
        for b in (-2, -1, 0, 1, 2):
            u, v = f32(cx), f32(cy)
            for _ in range(abs(a)):
                u = np.nextafter(u, f32(np.sign(a) * np.inf))
            for _ in range(abs(b)):
                v = np.nextafter(v, f32(np.sign(b) * np.inf))
            near.append((float(u), float(v)))
    rounding = rng.uniform(0.0, [W, H], (1000, 2)) + 1e-9 * rng.standard_normal((1000, 2))
    return {
        "grid": np.stack([gx.ravel(), gy.ravel()], axis=1),
        "wide": rng.uniform([-3.0 * W, -3.0 * H], [4.0 * W, 4.0 * H], (3000, 2)),
        "principal": np.array(near),
        "rounding": rounding,
        "nonfinite": NONFINITE.copy(),
    }


def all_points(cam: Cam, seed: int = 0) -> np.ndarray:
    return np.concatenate(list(point_sets(cam, seed).values()))


def cv2_undistort(cam: Cam, pts, output: str) -> np.ndarray:
    """The definition: cv2 on a float32 copy, P=None (normalised) or P=K (pixels); (n, 2) float32."""
    import cv2

    p = np.ascontiguousarray(pts, dtype=np.float32).reshape(-1, 1, 2)
    P = cam.K if output == "pixels" else None
    fn = cv2.fisheye.undistortPoints if cam.fisheye else cv2.undistortPoints
    return fn(p, cam.K, cam.d, P=P).reshape(-1, 2)


def branches(cam: Cam, pts) -> set[str]:
    """Which branches of the inverse map `pts` reach for `cam`:
    icdist_neg  pinhole: the rational factor turns negative at some iteration (cv2 restarts from the distorted point);
    sentinel    fisheye: cv2 returns (-1e6, -1e6) in normalised output (Newton failed or flipped theta's sign);
    theta_tiny  fisheye: 0 < theta_d <= 1e-8 (no Newton, scale 0) for a finite point;
    nonfinite   a NaN or infinite coordinate."""
    p = np.ascontiguousarray(pts, dtype=np.float32).astype(np.float64).reshape(-1, 2)
    out = set()
    if not np.isfinite(p).all():
        out.add("nonfinite")
    p = p[np.isfinite(p).all(axis=1)]
    fx, fy, cx, cy = cam.K[0, 0], cam.K[1, 1], cam.K[0, 2], cam.K[1, 2]
    x0, y0 = (p[:, 0] - cx) / fx, (p[:, 1] - cy) / fy
    if cam.fisheye:
        td = np.sqrt(x0 * x0 + y0 * y0)
        if ((td > 0) & (td <= 1e-8)).any():
            out.add("theta_tiny")
        if (cv2_undistort(cam, p, "normalized") == np.float32(SENTINEL)).all(axis=1).any():
            out.add("sentinel")
        return out
    k = np.zeros(12)
    k[: len(cam.d)] = cam.d
    x, y, live = x0.copy(), y0.copy(), np.ones(len(p), bool)
    for _ in range(5):
        r2 = x * x + y * y
        ic = (1 + ((k[7] * r2 + k[6]) * r2 + k[5]) * r2) / (1 + ((k[4] * r2 + k[1]) * r2 + k[0]) * r2)
        if (live & (ic < 0)).any():
            out.add("icdist_neg")
        live &= ic >= 0
        dx = 2 * k[2] * x * y + k[3] * (r2 + 2 * x * x) + k[8] * r2 + k[9] * r2 * r2
        dy = k[2] * (r2 + 2 * y * y) + 2 * k[3] * x * y + k[10] * r2 + k[11] * r2 * r2
        x, y = np.where(live, (x0 - dx) * ic, x0), np.where(live, (y0 - dy) * ic, y0)
    return out


def assert_same_f32(got, ref, what):
    """float32 equality with NaN positions equal (-0.0 == 0.0: cv2 itself returns -0. in places)."""
    got, ref = np.asarray(got, np.float32), np.asarray(ref, np.float32)
    assert got.shape == ref.shape, what
    assert np.array_equal(np.isnan(got), np.isnan(ref)), f"{what}: NaN positions differ"
    bad = ~np.isnan(ref) & (got != ref)
    assert not bad.any(), f"{what}: {bad.any(axis=1).sum()} of {len(ref)} rows differ, first {np.argwhere(bad)[0]}: " \
                          f"{got[bad.any(axis=1)][0]} vs {ref[bad.any(axis=1)][0]}"


def ulp32(a, b) -> np.ndarray:
    """Per-element float32 ulp distance of finite values (sign-magnitude mapped onto one integer line)."""
    def key(x):
        i = np.asarray(x, np.float32).view(np.int32).astype(np.int64)
        return np.where(i < 0, -(i & 0x7FFFFFFF), i)

    return np.abs(key(a) - key(b))
