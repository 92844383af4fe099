"""Synthetic multi-view scenes for the PatchMatch hot path: camera preparation + image rendering.

Host-side input preparation only (NumPy); nothing here is on the timed path.

* `prepare_cameras` restates the reference's camera preparation
  (cameraGeometryUtils.h:174-353: P -> K,R,t via RQ, re-base so that the reference camera is
  K[I|0], per-camera P, M_inv, C, R_orig_inv, fx/fy/alpha, baseline 0.54) without OpenCV, producing
  exactly the `Camera_cu` fields the hot path reads (SURVEY.md §8b).
* `select_views` restates main.cpp:430-499 (angle filter on the central viewing rays),
  deterministically (the reference shuffles with srand(time(0)), main.cpp:493).
* `render_scene` renders every view of a textured height field by per-pixel ray casting, so the
  images are photo-consistent and a true depth minimum exists; values are rounded to integers in
  [0, 255] exactly as the reference's 8-bit `imread` -> `convertTo(CV_32F)` inputs are
  (main.cpp:741-745, 939).
* `make_config(k)` builds the five BASELINE.json configurations.
"""
from __future__ import annotations

import dataclasses
import os
from dataclasses import dataclass, field, asdict
from typing import List, Optional, Sequence

import numpy as np

_DATA = os.path.join(os.path.dirname(os.path.abspath(__file__)), "data")

# cost combination (algorithmparameters.h:17)
COMB_ALL, COMB_BEST_N, COMB_ANGLE, COMB_GOOD = 0, 1, 2, 3


@dataclass
class AlgorithmParameters:
    """Mirror of the reference's AlgorithmParameters fields the device path reads
    (algorithmparameters.h:21-51; same names, same defaults)."""
    max_disparity: float = 256.0
    min_disparity: float = 0.0
    box_hsize: int = 19
    box_vsize: int = 19
    tau_color: float = 10.0
    tau_gradient: float = 2.0
    alpha: float = 0.9
    gamma: float = 10.0
    iterations: int = 8
    color_processing: bool = False
    good_factor: float = 1.5
    n_best: int = 2
    cost_comb: int = COMB_BEST_N
    depthMin: float = -1.0
    depthMax: float = -1.0
    min_angle: float = 5.0
    max_angle: float = 45.0
    max_views: int = 9


@dataclass
class Camera:
    """The Camera_cu fields (camera.h:7-62) as float32 arrays; matrices 3x3 row-major."""
    K: np.ndarray
    K_inv: np.ndarray
    R: np.ndarray
    R_orig_inv: np.ndarray
    M_inv: np.ndarray
    P: np.ndarray          # 3x4
    t: np.ndarray          # 3
    C: np.ndarray          # 3
    fx: float
    fy: float
    f: float
    alpha: float
    baseline: float = 0.54


@dataclass
class Scene:
    name: str
    rows: int
    cols: int
    images: np.ndarray                  # [n_images, rows, cols] float32, index 0 = reference
    cameras: List[Camera]
    subset: List[int]                   # viewSelectionSubset: indices into images/cameras
    params: AlgorithmParameters
    gt_depth: Optional[np.ndarray] = None   # [rows, cols] depth of the rendered surface in the ref view
    meta: dict = field(default_factory=dict)

    @property
    def n_views(self) -> int:
        return len(self.subset)


# ----------------------------------------------------------------------------------------------
# camera preparation
# ----------------------------------------------------------------------------------------------

def load_dtu_projections() -> np.ndarray:
    """[64,3,4] float64 DTU projection matrices (tools/make_dtu_fixture.py)."""
    return np.load(os.path.join(_DATA, "dtu_calib_P.npy"))


def rq3(M: np.ndarray):
    """RQ decomposition M = K @ R with K upper triangular (positive diagonal), R a rotation."""
    Q, U = np.linalg.qr(np.flipud(M).T)
    K = np.fliplr(np.flipud(U.T))
    R = np.flipud(Q.T)
    S = np.diag(np.where(np.diag(K) < 0, -1.0, 1.0))
    return K @ S, S @ R


def decompose_projection(P: np.ndarray):
    """P -> (K, R, C) with P ~ K [R | -R C]; the role cv::decomposeProjectionMatrix plays at
    cameraGeometryUtils.h:252."""
    P = np.asarray(P, dtype=np.float64)
    M = P[:, :3]
    if np.linalg.det(M) < 0:
        P = -P
        M = P[:, :3]
    K, R = rq3(M)
    C = -np.linalg.solve(M, P[:, 3])
    return K, R, C


def scale_K(K: np.ndarray, scale_factor: float) -> np.ndarray:
    """cameraGeometryUtils.h:136-147 (focal lengths and principal point divided by the factor)."""
    Ks = K.copy()
    Ks[0, 0] /= scale_factor
    Ks[1, 1] /= scale_factor
    Ks[0, 2] /= scale_factor
    Ks[1, 2] /= scale_factor
    return Ks


def _center_of(P: np.ndarray) -> np.ndarray:
    return -np.linalg.solve(P[:, :3], P[:, 3])


def prepare_cameras(Ps: Sequence[np.ndarray], cam_scale: float = 1.0) -> List[Camera]:
    """Projection matrices (index 0 = reference view) -> Camera_cu field values.
    Follows cameraGeometryUtils.h:251-346."""
    Ks, Rs, ts = [], [], []
    for P in Ps:
        K, R, C = decompose_projection(P)
        K = K / K[2, 2]
        Ks.append(K)
        Rs.append(R)
        ts.append(-R @ C)
    T0 = np.eye(4)
    T0[:3, :3] = Rs[0]
    T0[:3, 3] = ts[0]
    transform = np.linalg.inv(T0)                      # :282-283 reference -> origin
    Kref = scale_K(Ks[0], cam_scale)                   # :291 "assuming K is the same for all cameras"
    cams = []
    for K, R, t in zip(Ks, Rs, ts):
        T = np.eye(4)
        T[:3, :3] = R
        T[:3, 3] = t
        Tt = T @ transform                             # transformCamera, :117-134
        Pn = Kref @ Tt[:3, :4]
        Kc = scale_K(K, cam_scale)
        f32 = lambda a: np.ascontiguousarray(a, dtype=np.float32)
        cams.append(Camera(
            K=f32(Kc), K_inv=f32(np.linalg.inv(Kc)), R=f32(Tt[:3, :3]), R_orig_inv=f32(np.linalg.inv(R)),
            M_inv=f32(np.linalg.inv(Pn[:, :3])), P=f32(Pn), t=f32(Tt[:3, 3]), C=f32(_center_of(Pn)),
            fx=float(np.float32(Kref[0, 0])), fy=float(np.float32(Kref[1, 1])), f=float(np.float32(Kref[0, 0])),
            alpha=float(np.float32(Kref[0, 0]) / np.float32(Kref[1, 1])), baseline=0.54))
    return cams


def view_vector(cam: Camera, x: float, y: float) -> np.ndarray:
    """cameraGeometryUtils.h:68-77: unit ray through pixel (x, y)."""
    pt = np.array([x, y, 1.0]) - cam.P[:, 3].astype(np.float64)
    X = cam.M_inv.astype(np.float64) @ pt
    v = X - cam.C.astype(np.float64)
    return v / np.linalg.norm(v)


def view_angles(cams: Sequence[Camera], cols: int, rows: int) -> np.ndarray:
    """Angle (radians) between the central ray of camera 0 and of every camera (main.cpp:433-460)."""
    x, y = cols // 2, rows // 2
    v0 = view_vector(cams[0], x, y)
    out = np.zeros(len(cams))
    for i, c in enumerate(cams):
        d = float(np.clip(np.dot(v0, view_vector(c, x, y)), -1.0, 1.0))
        out[i] = np.arccos(d)
    return out


def select_views(cams: Sequence[Camera], cols: int, rows: int, params: AlgorithmParameters,
                 n_views: Optional[int] = None) -> List[int]:
    """main.cpp:430-499, deterministic: accept cameras whose central-ray angle to the reference lies
    in (min_angle, max_angle); keep the first `max_views` in index order (the reference picks a
    random subset).  With `n_views` set, return exactly that many: accepted cameras first (index
    order), then the remaining ones by increasing distance from the accepted angle band."""
    ang = np.degrees(view_angles(cams, cols, rows))
    ok = [i for i in range(1, len(cams)) if params.min_angle < ang[i] < params.max_angle]
    if n_views is None:
        return ok[: params.max_views] if len(ok) >= params.max_views else ok
    if len(ok) >= n_views:
        return ok[:n_views]
    rest = [i for i in range(1, len(cams)) if i not in ok]
    mid = 0.5 * (params.min_angle + params.max_angle)
    rest.sort(key=lambda i: abs(ang[i] - mid))
    sel = ok + rest[: n_views - len(ok)]
    if len(sel) < n_views:
        raise ValueError("not enough cameras: need %d source views, have %d" % (n_views, len(sel)))
    return sel


def synthetic_rig(n_src: int, K: np.ndarray, distance: float, min_deg: float, max_deg: float,
                  seed: int = 7) -> List[np.ndarray]:
    """Projection matrices for 1 reference + n_src source cameras on a spherical cap around the
    reference, all looking at the point `distance` in front of it; source cameras sit at polar angles
    in (min_deg, max_deg) from the reference's optical axis (golden-angle spiral in azimuth)."""
    target = np.array([0.0, 0.0, distance])
    Ps = [K @ np.hstack([np.eye(3), np.zeros((3, 1))])]
    rng = np.random.default_rng(seed)
    for k in range(n_src):
        pol = np.radians(min_deg + (max_deg - min_deg) * (0.08 + 0.84 * ((k * 0.618034) % 1.0)))
        az = 2.0 * np.pi * ((k * 0.381966 + 0.11) % 1.0)
        d = distance * (1.0 + 0.04 * rng.uniform(-1, 1))
        C = target + d * np.array([np.sin(pol) * np.cos(az), np.sin(pol) * np.sin(az), -np.cos(pol)])
        z = (target - C) / np.linalg.norm(target - C)
        up = np.array([0.0, 1.0, 0.0])
        x = np.cross(up, z)
        x /= np.linalg.norm(x)
        y = np.cross(z, x)
        R = np.stack([x, y, z])
        Ps.append(K @ np.hstack([R, (-R @ C)[:, None]]))
    return Ps


# ----------------------------------------------------------------------------------------------
# rendering
# ----------------------------------------------------------------------------------------------

class HeightField:
    """Surface Z = f(X, Y) in the re-based frame (reference camera = K[I|0]) with a procedural
    texture T(X, Y).  `unit` is the world length of one reference pixel at depth z0."""

    def __init__(self, z0: float, unit: float, seed: int = 1234, relief: float = 0.035, tilt=(0.10, -0.06), hard: bool = False):
        rng = np.random.default_rng(seed)
        self.z0, self.unit = float(z0), float(unit)
        # "hard" variant (bench.py --scene hard): raised blocks with vertical walls (depth discontinuities -> occlusions
        # between views), a texture-less band, and per-view sensor noise added by render_view
        self.hard = bool(hard)
        self.tilt = tilt
        self.relief = relief * z0
        self.bump_wl = np.array([260.0, 410.0, 690.0]) * unit        # long waves: gentle slopes
        self.bump_dir = rng.uniform(0, np.pi, 3)
        self.bump_ph = rng.uniform(0, 2 * np.pi, 3)
        self.tex_wl = np.array([5.0, 9.0, 17.0, 37.0, 71.0]) * unit
        self.tex_amp = np.array([22.0, 26.0, 24.0, 20.0, 16.0])
        self.tex_dir = rng.uniform(0, np.pi, 5)
        self.tex_ph = rng.uniform(0, 2 * np.pi, 5)
        self.lattice = rng.uniform(-1.0, 1.0, (256, 256)).astype(np.float32)
        self.cell = 4.0 * unit

    def height(self, X, Y):
        z = self.z0 + self.tilt[0] * X + self.tilt[1] * Y
        for wl, a, ph in zip(self.bump_wl, self.bump_dir, self.bump_ph):
            z = z + (self.relief / 3.0) * np.sin(2 * np.pi * (X * np.cos(a) + Y * np.sin(a)) / wl + ph)
        if self.hard:
            # blocks standing 6 % of z0 proud of the surface on a 520-pixel lattice, 170 pixels wide
            u = np.mod(X / (520.0 * self.unit) + 0.31, 1.0)
            w = np.mod(Y / (520.0 * self.unit) + 0.17, 1.0)
            z = z - 0.06 * self.z0 * ((u < 0.33) & (w < 0.33))
        return z

    def texture(self, X, Y):
        v = np.full(X.shape, 127.5, dtype=np.float64)
        for wl, amp, a, ph in zip(self.tex_wl, self.tex_amp, self.tex_dir, self.tex_ph):
            v += amp * np.sin(2 * np.pi * (X * np.cos(a) + Y * np.sin(a)) / wl + ph)
        u, w = X / self.cell, Y / self.cell
        iu, iw = np.floor(u), np.floor(w)
        fu, fw = u - iu, w - iw
        fu = fu * fu * (3 - 2 * fu)
        fw = fw * fw * (3 - 2 * fw)
        iu = iu.astype(np.int64)
        iw = iw.astype(np.int64)
        L = self.lattice
        a00 = L[iw & 255, iu & 255]
        a01 = L[iw & 255, (iu + 1) & 255]
        a10 = L[(iw + 1) & 255, iu & 255]
        a11 = L[(iw + 1) & 255, (iu + 1) & 255]
        v += 30.0 * ((a00 * (1 - fu) + a01 * fu) * (1 - fw) + (a10 * (1 - fu) + a11 * fu) * fw)
        if self.hard:
            # texture-less horizontal band: 140 reference pixels tall, constant grey
            band = np.abs(Y - 180.0 * self.unit) < 70.0 * self.unit
            v = np.where(band, 131.0, v)
        return v


def render_view(cam: Camera, rows: int, cols: int, hf: HeightField, iters: int = 10, band: int = 256, noise_seed: Optional[int] = None):
    """Ray-cast the height field for every pixel of `cam`; returns (image float32 with integer values
    in [0,255], depth along the camera's z axis).  `noise_seed`: add integer sensor noise in [-6, 6] (hard scenes)."""
    img = np.empty((rows, cols), dtype=np.float32)
    dep = np.empty((rows, cols), dtype=np.float32)
    Minv = cam.M_inv.astype(np.float64)
    C = cam.C.astype(np.float64)
    R = cam.R.astype(np.float64)
    t = cam.t.astype(np.float64)
    p4 = cam.P[:, 3].astype(np.float64)
    xs = np.arange(cols, dtype=np.float64)
    for y0 in range(0, rows, band):
        y1 = min(rows, y0 + band)
        ys = np.arange(y0, y1, dtype=np.float64)
        gx, gy = np.meshgrid(xs, ys)
        # a second point on each ray: X1 = M_inv (1*(x,y,1) - p4)  (get3Dpoint, depth 1)
        px = np.stack([gx - p4[0], gy - p4[1], np.full_like(gx, 1.0 - p4[2])], axis=-1)
        X1 = px @ Minv.T
        d = X1 - C
        lam = (hf.z0 - C[2]) / d[..., 2]
        for _ in range(iters):
            X = C[0] + lam * d[..., 0]
            Y = C[1] + lam * d[..., 1]
            lam = (hf.height(X, Y) - C[2]) / d[..., 2]
        X = C[0] + lam * d[..., 0]
        Y = C[1] + lam * d[..., 1]
        Z = C[2] + lam * d[..., 2]
        img[y0:y1] = np.clip(np.rint(hf.texture(X, Y)), 0, 255).astype(np.float32)
        dep[y0:y1] = (R[2, 0] * X + R[2, 1] * Y + R[2, 2] * Z + t[2]).astype(np.float32)
    if noise_seed is not None:
        noise = np.random.default_rng(noise_seed).integers(-6, 7, size=img.shape)
        img = np.clip(img + noise, 0, 255).astype(np.float32)
    return img, dep


def _render_job(job):
    cam, rows, cols, hf_args, noise_seed = job
    return render_view(cam, rows, cols, HeightField(**hf_args), noise_seed=noise_seed)


def ref0_frame(Ps: Sequence[np.ndarray]):
    """(R0, t0): a point X of the frame of the projections Ps is R0 X + t0 in the frame re-based on camera 0, where
    prepare_cameras puts the cameras and HeightField its surface."""
    _, R, C = decompose_projection(Ps[0])
    return R, -R @ C


def render_norm4(Ps: Sequence[np.ndarray], cam_scale: float, rows: int, cols: int, hf: HeightField, iters: int = 10,
                 band: int = 256) -> np.ndarray:
    """Ground truth of every camera in the layout of the pipeline's output (gpm_batch_run's out_norm4): [n, rows, cols, 4]
    float32, unit surface normal in the frame of Ps, facing the camera, and depth along the camera's z axis.  The ray cast
    of render_view does not converge on oblique rays; pixels whose ray ends more than 1e-6 z0 off the surface get depth 0
    (invalid), so every valid depth is on the surface."""
    cams = prepare_cameras(Ps, cam_scale)
    R0, _ = ref0_frame(Ps)
    out = np.empty((len(cams), rows, cols, 4), dtype=np.float32)
    eps = 0.01 * hf.unit
    xs = np.arange(cols, dtype=np.float64)
    for i, cam in enumerate(cams):
        Minv, C, p4 = cam.M_inv.astype(np.float64), cam.C.astype(np.float64), cam.P[:, 3].astype(np.float64)
        R, t = cam.R.astype(np.float64), cam.t.astype(np.float64)
        for y0 in range(0, rows, band):                        # the ray cast of render_view
            gx, gy = np.meshgrid(xs, np.arange(y0, min(rows, y0 + band), dtype=np.float64))
            d = np.stack([gx - p4[0], gy - p4[1], np.full_like(gx, 1.0 - p4[2])], axis=-1) @ Minv.T - C
            lam = (hf.z0 - C[2]) / d[..., 2]
            for _ in range(iters):
                lam = (hf.height(C[0] + lam * d[..., 0], C[1] + lam * d[..., 1]) - C[2]) / d[..., 2]
            X, Y, Z = C[0] + lam * d[..., 0], C[1] + lam * d[..., 1], C[2] + lam * d[..., 2]
            n = np.stack([(hf.height(X + eps, Y) - hf.height(X - eps, Y)) / (2 * eps),
                          (hf.height(X, Y + eps) - hf.height(X, Y - eps)) / (2 * eps), -np.ones_like(X)], axis=-1)
            n /= np.linalg.norm(n, axis=-1, keepdims=True)
            out[i, y0:y0 + len(X), :, :3] = n @ R0                    # R0^T n: back to the frame of Ps
            dep = R[2, 0] * X + R[2, 1] * Y + R[2, 2] * Z + t[2]
            on_surface = np.abs(Z - hf.height(X, Y)) <= 1e-6 * hf.z0
            out[i, y0:y0 + len(X), :, 3] = np.where(on_surface & (np.abs(dep) < 1e30), dep, 0.0)
    return out


def gt_points(Ps: Sequence[np.ndarray], cam_scale: float, rows: int, cols: int, hf: HeightField, stride: int = 1,
              norm4: Optional[np.ndarray] = None) -> np.ndarray:
    """Ground-truth point cloud of a height-field scene: the surface the cameras see.  Every valid pixel (depth > 0) of the
    maps of render_norm4, taking every `stride`-th row and column, back-projected in float64 with get3Dpoint
    (X = M_inv (d (x, y, 1) - P_col34)) through the fusion's camera of its view (DESIGN.md §12), so the points are in the
    un-rebased world frame of gpm_fuse's vertices.  The maps were ray cast through the float32 camera fields of
    prepare_cameras, so a point lies off the surface by up to about 3e-5 z0 (the fusion's vertices inherit the same).
    `norm4`: those maps, if already rendered.  Returns (N, 3) float32 in (view, y, x) order.  It stands in for a dataset's
    observation mask."""
    if norm4 is None:
        norm4 = render_norm4(Ps, cam_scale, rows, cols, hf)
    ys, xs = np.mgrid[0:rows:stride, 0:cols:stride].astype(np.float64)
    out = []
    for P, n4 in zip(Ps, norm4):
        K, R, C = decompose_projection(P)
        Pv = scale_K(K / K[2, 2], cam_scale) @ np.hstack([R, (-R @ C)[:, None]])
        d = n4[::stride, ::stride, 3].astype(np.float64)
        ok = d > 0
        h = np.stack([d[ok] * xs[ok], d[ok] * ys[ok], d[ok]], axis=1) - Pv[:, 3]
        out.append(h @ np.linalg.inv(Pv[:, :3]).T)
    return np.ascontiguousarray(np.concatenate(out), dtype=np.float32)


def render_scene(name: str, Ps: Sequence[np.ndarray], rows: int, cols: int, params: AlgorithmParameters,
                 cam_scale: float = 1.0, n_views: Optional[int] = None, z0: Optional[float] = None,
                 seed: int = 1234, only_selected: bool = True, hard: bool = False, workers: int = 0,
                 render_positions: Optional[Sequence[int]] = None) -> Scene:
    """Prepare cameras, select views, render the reference and the selected source views, and
    derive min/max_disparity from the depth range as main.cpp:898-906 does.
    `render_positions`: positions in the view subset to render (others stay zero) — a view-shard rank only needs the
    reference image and its own views; `workers` > 1 renders the views in a fork pool (same bits)."""
    cams = prepare_cameras(Ps, cam_scale)
    subset = select_views(cams, cols, rows, params, n_views)
    keep = [0] + subset if only_selected else list(range(len(cams)))
    cams = [cams[i] for i in keep]
    subset = list(range(1, len(keep))) if only_selected else subset
    z0 = 0.5 * (params.depthMin + params.depthMax) if z0 is None else z0
    hf_args = dict(z0=z0, unit=z0 / cams[0].fx, seed=seed, hard=hard)
    images = np.zeros((len(cams), rows, cols), dtype=np.float32)
    wanted = list(range(len(cams)))
    if render_positions is not None and only_selected:
        wanted = [0] + [1 + p for p in sorted(set(render_positions))]      # cams = [reference] + subset in order
    jobs = [(cams[i], rows, cols, hf_args, (seed * 1000003 + 7919 * i) if hard else None) for i in wanted]
    if workers > 1 and len(jobs) > 1:
        import multiprocessing as mp
        with mp.get_context("fork").Pool(min(workers, len(jobs))) as pool:
            results = pool.map(_render_job, jobs, chunksize=1)
    else:
        results = [_render_job(j) for j in jobs]
    gt = None
    for i, (img, d) in zip(wanted, results):
        images[i] = img
        if i == 0:
            gt = d
    f = np.float32(cams[0].f)
    b = np.float32(cams[0].baseline)
    params.min_disparity = float(f * b / np.float32(params.depthMax))     # main.cpp:905
    params.max_disparity = float(f * b / np.float32(params.depthMin))     # main.cpp:906
    return Scene(name=name + ("_hard" if hard else ""), rows=rows, cols=cols, images=images, cameras=cams, subset=subset, params=params,
                 gt_depth=gt, meta={"z0": z0, "seed": seed, "cam_scale": cam_scale, "hard": hard,
                                    "rendered": wanted})


def colorize(scene: Scene) -> Scene:
    """The same scene with float4 images [n, rows, cols, 4] and color_processing on (the reference converts the
    8-bit BGR image to 4 float channels, main.cpp:560-605 / 1080-1110; the 4th channel is never read by the float4
    operators, vector_operations.h:3-38).  Each channel is a fixed function of the rendered gray value, so the views
    stay photo-consistent; values are integers in [0, 255] like a decoded 8-bit image."""
    g = scene.images.astype(np.float64)
    b = g
    gr = np.clip(np.rint(245.0 - 0.85 * g), 0, 255)
    r = np.clip(np.rint(127.5 + 110.0 * np.sin(g / 23.0)), 0, 255)
    images = np.stack([b, gr, r, np.zeros_like(g)], axis=-1).astype(np.float32)
    params = dataclasses.replace(scene.params, color_processing=True)
    return dataclasses.replace(scene, name=scene.name + "_color", images=np.ascontiguousarray(images), params=params)


# ----------------------------------------------------------------------------------------------
# BASELINE.json configurations
# ----------------------------------------------------------------------------------------------

DTU_REF_POSITION = 24          # 0-based index of DTU position 25 (SURVEY.md §8d)


def _dtu_Ps() -> List[np.ndarray]:
    P = load_dtu_projections()
    order = [DTU_REF_POSITION] + [i for i in range(P.shape[0]) if i != DTU_REF_POSITION]
    return [P[i] for i in order]


def make_config(k: int, rows: Optional[int] = None, cols: Optional[int] = None,
                n_views: Optional[int] = None, iterations: Optional[int] = None, seed: int = 1234,
                hard: bool = False, workers: int = 0, render_positions: Optional[Sequence[int]] = None) -> Scene:
    """The five BASELINE.json configurations (SURVEY.md §8 table) and, as k = 6, north_star's strong-scaling workload
    (1600x1200, 60 source views, dtu_fast parameters).  `rows`/`cols`/`n_views`/`iterations` override the configuration
    (used by tests to shrink a case; K is scaled with the image so the geometry stays the same); `hard` adds occluding
    blocks, a texture-less band and sensor noise; `workers` / `render_positions` see render_scene."""
    kw = dict(hard=hard, workers=workers, render_positions=render_positions)
    if k == 1:      # 320x240, 2 source views, 3 iterations, blocksize 15 — plumbing / parity
        W, H, V, it, b, nb = 320, 240, 2, 3, 15, 2
    elif k == 2:    # dtu_fast: blocksize 15, n_best 3, depth 300-800, angles 10-30 (scripts/dtu_fast.sh:10-21)
        W, H, V, it, b, nb = 1600, 1200, 10, 8, 15, 3
    elif k == 3:    # dtu_accurate: blocksize 25 (scripts/dtu_accurate.sh:10-20)
        W, H, V, it, b, nb = 1600, 1200, 30, 8, 25, 3
    elif k == 4:    # templeRing: blocksize 11, depth 0.3-0.8, angles 5-45 (scripts/templeRing.sh:9-24)
        W, H, V, it, b, nb = 640, 480, 47, 8, 11, 3
    elif k == 5:    # synthetic 3200x2400, 64 views
        W, H, V, it, b, nb = 3200, 2400, 64, 8, 15, 3
    elif k == 6:    # north_star: "1600x1200 ... 60 source views", DTU shape, dtu_fast parameters (view-shard workload)
        W, H, V, it, b, nb = 1600, 1200, 60, 8, 15, 3
    else:
        raise ValueError("config must be 1..6")
    cols_ = W if cols is None else cols
    rows_ = H if rows is None else rows
    V = V if n_views is None else n_views
    it = it if iterations is None else iterations
    prm = AlgorithmParameters(box_hsize=b, box_vsize=b, iterations=it, n_best=nb, cost_comb=COMB_BEST_N, gamma=10.0)
    if k == 4:
        prm.depthMin, prm.depthMax, prm.min_angle, prm.max_angle = 0.3, 0.8, 5.0, 45.0
        K = np.array([[1520.4, 0, 302.32], [0, 1525.9, 246.87], [0, 0, 1.0]])
        scale = 640.0 / cols_
        Ps = synthetic_rig(V, K, distance=0.55, min_deg=5.0, max_deg=45.0, seed=seed)
        return render_scene("cfg4_temple_ring", Ps, rows_, cols_, prm, cam_scale=scale, n_views=V, seed=seed, **kw)
    prm.depthMin, prm.depthMax, prm.min_angle, prm.max_angle = 300.0, 800.0, 10.0, 30.0
    if k == 5:
        K0, _, _ = decompose_projection(load_dtu_projections()[DTU_REF_POSITION])
        K0 = K0 / K0[2, 2]
        scale = 1600.0 / cols_          # 0.5 at 3200x2400: K x 2 (scaleK divides by the factor)
        Ps = synthetic_rig(V, K0, distance=550.0, min_deg=10.0, max_deg=30.0, seed=seed)
        return render_scene("cfg5_synth_64v", Ps, rows_, cols_, prm, cam_scale=scale, n_views=V, seed=seed, **kw)
    scale = 1600.0 / cols_
    name = {1: "cfg1_plumbing", 2: "cfg2_dtu_fast", 3: "cfg3_dtu_accurate", 6: "dtu60_view_shard"}[k]
    return render_scene(name, _dtu_Ps(), rows_, cols_, prm, cam_scale=scale, n_views=V, seed=seed, **kw)


def params_as_dict(p: AlgorithmParameters) -> dict:
    return asdict(p)
