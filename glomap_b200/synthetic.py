"""Deterministic synthetic scenes of the shapes BASELINE.json names.

The reference synthesises its test data with ``colmap::SynthesizeDataset``
(glomap/controllers/global_mapper_test.cc:58-64), which is not vendored; these
generators produce the same kind of world (cameras looking at a point cloud,
pixel observations with optional noise, a view graph with relative rotations)
directly in the flat SoA layout that crosses the C ABI (include/b200sfm.h).

Shapes (SURVEY.md 8(d)):
  config 1: ring of 100 cameras, 500 relative poses        -> make_ring_relposes
  config 2: 1k cams / 200k points / 2M observations         -> make_scene(1000, 200000)
  config 4: 10k cams / 2M points / 20M observations         -> make_scene(10000, 2000000)
  config 5: 100k-camera lattice view graph, 5M edges        -> make_lattice_view_graph
"""
from __future__ import annotations

import dataclasses

import numpy as np

from . import geometry as geo

# COLMAP camera model ids (colmap/sensor/models.h; un-vendored, public enum).
SIMPLE_PINHOLE, PINHOLE, SIMPLE_RADIAL, RADIAL = 0, 1, 2, 3
INTR_STRIDE = 12  # doubles reserved per intrinsics block across the C ABI
MODEL_NUM_PARAMS = {SIMPLE_PINHOLE: 3, PINHOLE: 4, SIMPLE_RADIAL: 4, RADIAL: 5}


@dataclasses.dataclass
class Scene:
    """Flat BA/GP problem: CSR by point (track) over observations."""
    quat: np.ndarray          # [C,4] xyzw cam_from_world
    trans: np.ndarray         # [C,3]
    points: np.ndarray        # [P,3]
    pt_obs_begin: np.ndarray  # [P+1] int64
    obs_cam: np.ndarray       # [N] int32
    obs_xy: np.ndarray        # [N,2] pixels
    cam_intr: np.ndarray      # [C] int32 -> intrinsics block
    intr_model: np.ndarray    # [K] int32
    intr_params: np.ndarray   # [K, INTR_STRIDE]

    @property
    def C(self):
        return len(self.quat)

    @property
    def P(self):
        return len(self.points)

    @property
    def N(self):
        return len(self.obs_cam)

    def copy(self):
        return Scene(*[np.array(getattr(self, f.name), copy=True) for f in dataclasses.fields(self)])


def project(model: int, params: np.ndarray, Xc: np.ndarray) -> np.ndarray:
    """Pixel projection of camera-frame points for the supported COLMAP models
    (SIMPLE_PINHOLE f,cx,cy | PINHOLE fx,fy,cx,cy | SIMPLE_RADIAL f,cx,cy,k |
    RADIAL f,cx,cy,k1,k2)."""
    u = Xc[..., 0] / Xc[..., 2]
    v = Xc[..., 1] / Xc[..., 2]
    if model == SIMPLE_PINHOLE:
        f, cx, cy = params[:3]
        return np.stack([f * u + cx, f * v + cy], -1)
    if model == PINHOLE:
        fx, fy, cx, cy = params[:4]
        return np.stack([fx * u + cx, fy * v + cy], -1)
    r2 = u * u + v * v
    if model == SIMPLE_RADIAL:
        f, cx, cy, k = params[:4]
        d = 1 + k * r2
    elif model == RADIAL:
        f, cx, cy, k1, k2 = params[:5]
        d = 1 + k1 * r2 + k2 * r2 * r2
    else:
        raise ValueError(f"unsupported camera model {model}")
    return np.stack([f * u * d + cx, f * v * d + cy], -1)


def _look_at_rotations(centers: np.ndarray, rng, jitter_deg: float) -> np.ndarray:
    """cam_from_world rotations with the optical axis (+z) toward the origin,
    plus a random rotation of up to ``jitter_deg`` degrees."""
    z = -centers / np.linalg.norm(centers, axis=1, keepdims=True)
    up = np.tile(np.array([0.0, 1.0, 0.0]), (len(centers), 1))
    bad = np.abs((z * up).sum(1)) > 0.99
    up[bad] = np.array([1.0, 0.0, 0.0])
    x = np.cross(up, z)
    x /= np.linalg.norm(x, axis=1, keepdims=True)
    y = np.cross(z, x)
    R = np.stack([x, y, z], axis=1)  # rows = camera axes in world coords
    if jitter_deg > 0:
        w = rng.normal(size=(len(centers), 3))
        w /= np.linalg.norm(w, axis=1, keepdims=True)
        w *= np.radians(jitter_deg) * rng.uniform(0, 1, size=(len(centers), 1))
        R = geo.so3_exp(w) @ R
    return R


def make_cameras(C: int, seed: int = 1, jitter_deg: float = 10.0):
    """Camera poses only (identical on every rank)."""
    rng = np.random.default_rng([seed, 0])
    d = rng.normal(size=(C, 3))
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    centers = d * rng.uniform(8, 12, size=(C, 1))
    R = _look_at_rotations(centers, rng, jitter_deg)
    t = -np.einsum("nij,nj->ni", R, centers)
    return R, t


def make_intrinsics(C: int, model, focal: float, image_size: int, num_intrinsics: int):
    """``model``: one camera model for every block, or a sequence of models that block k takes cyclically
    (model[k % len(model)]), as a database with several kinds of camera has."""
    K = num_intrinsics
    models = np.atleast_1d(np.asarray(model, dtype=np.int32))
    intr_model = models[np.arange(K) % len(models)]
    intr_params = np.zeros((K, INTR_STRIDE))
    half = image_size / 2
    for k in range(K):
        # a few shared blocks: 2 % steps around `focal`; many (per-image) blocks: bounded +-10 % variation
        f = focal * (1 + 0.02 * (k - (K - 1) / 2)) if K <= 8 else focal * (1 + 0.1 * np.sin(1.7 * k))
        model = int(intr_model[k])
        if model == SIMPLE_PINHOLE:
            intr_params[k, :3] = [f, half, half]
        elif model == PINHOLE:
            intr_params[k, :4] = [f, f * 1.01, half, half]
        elif model == SIMPLE_RADIAL:
            intr_params[k, :4] = [f, half, half, 0.02]
        elif model == RADIAL:
            intr_params[k, :5] = [f, half, half, 0.02, -0.005]
        else:
            raise ValueError(f"unsupported camera model {model}")
    cam_intr = (np.arange(C) % K).astype(np.int32)
    return cam_intr, intr_model, intr_params


def make_scene(C: int, P: int, mean_track_len: float = 10.0, seed: int = 1, pixel_sigma: float = 0.0,
               model: int = SIMPLE_PINHOLE, focal: float = 1000.0, image_size: int = 1000,
               num_intrinsics: int = 1, candidates_mult: int = 3, ragged: bool = True,
               jitter_deg: float = 10.0, chunk: int = 100_000, point_range: tuple[int, int] | None = None) -> Scene:
    """Cameras on a shell r in [8,12] looking at the origin (+-jitter), points
    uniform in a ball of radius 3, each point observed by the cameras (of a
    random candidate set) with the smallest off-axis angle.  Track lengths are
    3 + Poisson(mean-3) when ``ragged`` else constant.

    Points are generated in chunks of ``chunk`` with one RNG stream per chunk,
    so ``point_range=(a, b)`` (multiples of ``chunk``) yields exactly the
    points [a, b) of the full scene -- how the multi-GPU bench shards."""
    R, t = make_cameras(C, seed, jitter_deg)
    cam_intr, intr_model, intr_params = make_intrinsics(C, model, focal, image_size, num_intrinsics)
    K = num_intrinsics
    a, b = point_range if point_range is not None else (0, P)
    assert a % chunk == 0 and (b % chunk == 0 or b == P), "point_range must align with chunk"
    M = int(min(C, max(int(candidates_mult * mean_track_len), 8)))
    R32, t32 = R.astype(np.float32), t.astype(np.float32)
    tan_half = 0.48 * image_size / focal

    pts_chunks, obs_cam_chunks, obs_xy_chunks, len_chunks = [], [], [], []
    for s in range(a, b, chunk):
        e = min(P, s + chunk)
        n = e - s
        rng = np.random.default_rng([seed, 1 + s // chunk])
        pts = rng.normal(size=(n, 3))
        pts /= np.linalg.norm(pts, axis=1, keepdims=True)
        pts *= 3.0 * rng.uniform(0, 1, size=(n, 1)) ** (1 / 3)
        if ragged:
            lens = 3 + rng.poisson(max(mean_track_len - 3, 0), size=n)
        else:
            lens = np.full(n, int(round(mean_track_len)))
        lens = np.minimum(lens, M).astype(np.int64)
        if M >= C:
            cand = np.tile(np.arange(C), (n, 1))
        else:
            cand = rng.integers(0, C, size=(n, M))
            cand.sort(axis=1)
        dup = np.zeros_like(cand, dtype=bool)
        dup[:, 1:] = cand[:, 1:] == cand[:, :-1]
        # candidate scoring in float32 (only the ranking matters)
        Xc = np.einsum("nmij,nj->nmi", R32[cand], pts.astype(np.float32)) + t32[cand]
        z = Xc[..., 2]
        cosang = z / np.linalg.norm(Xc, axis=-1)
        with np.errstate(divide="ignore", invalid="ignore"):
            u = Xc[..., 0] / z
            v = Xc[..., 1] / z
        vis = (z > 0.1) & (np.abs(u) < tan_half) & (np.abs(v) < tan_half) & ~dup
        score = np.where(vis, -cosang, np.inf)
        order = np.argsort(score, axis=1, kind="stable")
        ln = np.minimum(lens, vis.sum(1))
        take = np.arange(M)[None, :] < ln[:, None]
        sel_cam = np.take_along_axis(cand, order, axis=1)[take]
        pidx = np.repeat(np.arange(n), ln)
        Xs = np.einsum("nij,nj->ni", R[sel_cam], pts[pidx]) + t[sel_cam]
        xy = np.empty((len(sel_cam), 2))
        ci = cam_intr[sel_cam]
        for k in range(K):
            mk = ci == k if K > 1 else slice(None)
            xy[mk] = project(int(intr_model[k]), intr_params[k], Xs[mk])
        if pixel_sigma > 0:
            xy += rng.normal(scale=pixel_sigma, size=xy.shape)
        pts_chunks.append(pts)
        obs_cam_chunks.append(sel_cam.astype(np.int32))
        obs_xy_chunks.append(xy)
        len_chunks.append(ln)
    points = np.concatenate(pts_chunks)
    obs_cam = np.concatenate(obs_cam_chunks)
    obs_xy = np.concatenate(obs_xy_chunks)
    final_lens = np.concatenate(len_chunks)
    pt_obs_begin = np.zeros(len(points) + 1, dtype=np.int64)
    np.cumsum(final_lens, out=pt_obs_begin[1:])
    quat = geo.rotmat_to_quat_xyzw_fast(R)
    return Scene(quat, t, points, pt_obs_begin, obs_cam, obs_xy, cam_intr, intr_model, intr_params)


def perturb_scene(scene: Scene, rot_deg: float = 0.5, center_frac: float = 0.01, point_frac: float = 0.01,
                  seed: int = 2, extent: float = 10.0, chunk: int = 100_000, point_offset: int = 0) -> Scene:
    """BA initial state: ground truth perturbed by ``rot_deg`` degrees,
    ``center_frac``*extent camera-centre noise, ``point_frac``*3 point noise
    (SURVEY.md 8(d) config 4).  Point noise uses one RNG stream per chunk of
    the global point index (``point_offset`` = first global index of a shard)."""
    rng = np.random.default_rng([seed, 0])
    out = scene.copy()
    R = geo.quat_xyzw_to_rotmat(scene.quat)
    c = geo.centers_from_pose(R, scene.trans)
    w = rng.normal(size=(scene.C, 3)) * np.radians(rot_deg) / np.sqrt(3)
    Rn = geo.so3_exp(w) @ R
    cn = c + rng.normal(size=c.shape) * center_frac * extent / np.sqrt(3)
    out.quat = geo.rotmat_to_quat_xyzw_fast(Rn)
    out.trans = -np.einsum("nij,nj->ni", Rn, cn)
    assert point_offset % chunk == 0
    for s in range(0, scene.P, chunk):
        e = min(scene.P, s + chunk)
        prng = np.random.default_rng([seed, 1 + (point_offset + s) // chunk])
        out.points[s:e] = scene.points[s:e] + prng.normal(size=(e - s, 3)) * point_frac * 3.0 / np.sqrt(3)
    return out


@dataclasses.dataclass
class RigScene:
    """Flat BA/GP problem with camera rigs (b200sfm_ba_problem_create_rig): the pose unknowns are
    the F frames (rig_from_world); an image is a frame seen through one sensor, whose cam_from_rig and
    intrinsics block are constants of the sensor (glomap/scene/frame.h, colmap::Rig).

    The image table (``image_frame`` / ``image_sensor``, image k = row k) and the rigs (``frame_rig``, ``sensor_rig``,
    ``rig_ref_sensor``) describe which sensors a frame uses; ``sensor_known`` marks the sensors whose cam_from_rig is
    known (a rig's reference sensor is, with the identity).  Left as None they default to the dense layout: one rig of
    all S sensors, sensor 0 its reference, every sensor known and image f * S + s = (frame f, sensor s)."""
    quat: np.ndarray          # [F,4] xyzw rig_from_world
    trans: np.ndarray         # [F,3]
    points: np.ndarray        # [P,3]
    pt_obs_begin: np.ndarray  # [P+1] int64
    obs_frame: np.ndarray     # [N] int32
    obs_sensor: np.ndarray    # [N] uint16
    obs_xy: np.ndarray        # [N,2] pixels
    sensor_quat: np.ndarray   # [S,4] xyzw cam_from_rig
    sensor_trans: np.ndarray  # [S,3] (NaN rows: translation not estimated yet)
    sensor_intr: np.ndarray   # [S] int32 -> intrinsics block
    intr_model: np.ndarray    # [K] int32
    intr_params: np.ndarray   # [K, INTR_STRIDE]
    image_frame: np.ndarray | None = None     # [I] int32 frame of every image
    image_sensor: np.ndarray | None = None    # [I] int32 sensor of every image
    frame_rig: np.ndarray | None = None       # [F] int32
    sensor_rig: np.ndarray | None = None      # [S] int32
    rig_ref_sensor: np.ndarray | None = None  # [R] int32 reference sensor of every rig
    sensor_known: np.ndarray | None = None    # [S] bool cam_from_rig known

    def __post_init__(self):
        F, S = len(self.quat), len(self.sensor_quat)
        if self.image_frame is None:
            self.image_frame = np.repeat(np.arange(F), S).astype(np.int32)
        if self.image_sensor is None:
            self.image_sensor = np.tile(np.arange(S), F).astype(np.int32)
        if self.frame_rig is None:
            self.frame_rig = np.zeros(F, np.int32)
        if self.sensor_rig is None:
            self.sensor_rig = np.zeros(S, np.int32)
        if self.rig_ref_sensor is None:
            self.rig_ref_sensor = np.zeros(1, np.int32)
        if self.sensor_known is None:
            self.sensor_known = np.ones(S, bool)

    @property
    def I(self):  # noqa: E743
        return len(self.image_frame)

    @property
    def sensor_is_ref(self):
        """[S] bool: the reference sensor of its rig (the sensors optimize_rig_poses keeps constant)."""
        ref = np.zeros(self.S, bool)
        r = np.asarray(self.rig_ref_sensor, np.int64)
        ref[r[r >= 0]] = True
        return ref

    def image_index(self):
        """[F, S] image of (frame, sensor), -1 where the table has none."""
        idx = np.full((self.F, self.S), -1, np.int64)
        idx[self.image_frame, self.image_sensor] = np.arange(self.I)
        return idx

    def obs_image(self):
        """[N] image of every observation."""
        return self.image_index()[self.obs_frame, self.obs_sensor]

    @property
    def C(self):
        return len(self.quat)

    @property
    def F(self):
        return len(self.quat)

    @property
    def S(self):
        return len(self.sensor_quat)

    @property
    def P(self):
        return len(self.points)

    @property
    def N(self):
        return len(self.obs_frame)

    def copy(self):
        return RigScene(*[np.array(getattr(self, f.name), copy=True) for f in dataclasses.fields(self)])

    def image_poses(self):
        """cam_from_world of the images of the table (dense layout: image id = f * S + s)."""
        Rf = geo.quat_xyzw_to_rotmat(self.quat)[self.image_frame]
        Rs = geo.quat_xyzw_to_rotmat(self.sensor_quat)[self.image_sensor]
        R = np.einsum("nij,njk->nik", Rs, Rf)
        t = np.einsum("nij,nj->ni", Rs, self.trans[self.image_frame]) + self.sensor_trans[self.image_sensor]
        return R, t

    def images_scene(self) -> Scene:
        """The same observations as a trivial-frame Scene over the images of the table (poses composed)."""
        R, t = self.image_poses()
        return Scene(geo.rotmat_to_quat_xyzw_fast(R), t, self.points.copy(), self.pt_obs_begin.copy(),
                     self.obs_image().astype(np.int32), self.obs_xy.copy(), self.sensor_intr[self.image_sensor].astype(np.int32),
                     self.intr_model.copy(), self.intr_params.copy())

    def rig_dict(self):
        """The ``rig`` argument of oracle.ba_oracle (per-image arrays over the image table)."""
        # img_sensor / sensor_q / sensor_t are read only with optimize_rig_poses (reference sensors: constant)
        sen = self.image_sensor
        return dict(obs_img=self.obs_image(), img_q=self.sensor_quat[sen].copy(), img_t=self.sensor_trans[sen].copy(),
                    img_intr=self.sensor_intr[sen].copy(), img_sensor=np.where(self.sensor_is_ref[sen], -1, sen),
                    sensor_q=self.sensor_quat.copy(), sensor_t=self.sensor_trans.copy())


def make_rig_scene(F: int, S: int, P: int, mean_track_len: float = 8.0, seed: int = 1, pixel_sigma: float = 0.0,
                   model: int = SIMPLE_PINHOLE, focal: float = 1000.0, image_size: int = 1000,
                   shared_intrinsics: bool = False, sensor_rot_deg: float = 20.0, sensor_offset: float = 0.4) -> RigScene:
    """F rigs of S cameras looking at a ball of points.  Sensor 0 is the reference sensor (identity
    cam_from_rig); the others are rotated by up to ``sensor_rot_deg`` and shifted by ``sensor_offset``.
    Every sensor has its own intrinsics block unless ``shared_intrinsics``; ``model`` may list one model per sensor
    (make_intrinsics).  Small sizes only (tests)."""
    rng = np.random.default_rng([seed, 77])
    Rf, tf = make_cameras(F, seed=seed, jitter_deg=5.0)
    w = rng.normal(size=(S, 3))
    w = w / np.linalg.norm(w, axis=1, keepdims=True) * np.radians(sensor_rot_deg) * rng.uniform(0.3, 1.0, size=(S, 1))
    w[0] = 0.0
    Rs = geo.so3_exp(w)
    ts = rng.normal(size=(S, 3))
    ts = ts / np.linalg.norm(ts, axis=1, keepdims=True) * sensor_offset
    ts[0] = 0.0
    K = 1 if shared_intrinsics else S
    _, intr_model, intr_params = make_intrinsics(S, model, focal, image_size, K)
    sensor_intr = (np.arange(S) % K).astype(np.int32)
    scene = RigScene(geo.rotmat_to_quat_xyzw_fast(Rf), tf, np.zeros((P, 3)), np.zeros(P + 1, np.int64),
                     np.zeros(0, np.int32), np.zeros(0, np.uint16), np.zeros((0, 2)), geo.rotmat_to_quat_xyzw_fast(Rs), ts,
                     sensor_intr, intr_model, intr_params)
    Ri, ti = scene.image_poses()
    d = rng.normal(size=(P, 3))
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    points = d * 3.0 * rng.uniform(0, 1, size=(P, 1)) ** (1 / 3)
    lens = 3 + rng.poisson(max(mean_track_len - 3, 0.0), size=P)
    fr, se, xy, begin = [], [], [], [0]
    lim = 0.5 * image_size / focal * 1.2
    for p in range(P):
        Xc = np.einsum("nij,j->ni", Ri, points[p]) + ti
        u, v = Xc[:, 0] / Xc[:, 2], Xc[:, 1] / Xc[:, 2]
        ok = np.nonzero((Xc[:, 2] > 0.5) & (np.abs(u) < lim) & (np.abs(v) < lim))[0]
        pick = rng.permutation(ok)[: lens[p]]
        pick.sort()
        for img in pick:
            f, sidx = divmod(int(img), S)
            k = sensor_intr[sidx]
            px = project(int(intr_model[k]), intr_params[k], Xc[img])
            fr.append(f); se.append(sidx); xy.append(px)
        begin.append(len(fr))
    scene.points = points
    scene.pt_obs_begin = np.asarray(begin, np.int64)
    scene.obs_frame = np.asarray(fr, np.int32)
    scene.obs_sensor = np.asarray(se, np.uint16)
    scene.obs_xy = np.asarray(xy, np.float64).reshape(-1, 2)
    if pixel_sigma > 0:
        scene.obs_xy = scene.obs_xy + rng.normal(size=scene.obs_xy.shape) * pixel_sigma
    return scene


def perturb_rig_scene(scene: RigScene, rot_deg: float = 0.5, center_frac: float = 0.01, point_frac: float = 0.01,
                      seed: int = 2, extent: float = 10.0) -> RigScene:
    """BA initial state for a rig scene: frame poses and points perturbed like ``perturb_scene``."""
    rng = np.random.default_rng([seed, 5])
    out = scene.copy()
    R = geo.quat_xyzw_to_rotmat(scene.quat)
    c = geo.centers_from_pose(R, scene.trans)
    w = rng.normal(size=(scene.F, 3)) * np.radians(rot_deg) / np.sqrt(3)
    Rn = geo.so3_exp(w) @ R
    cn = c + rng.normal(size=c.shape) * center_frac * extent / np.sqrt(3)
    out.quat = geo.rotmat_to_quat_xyzw_fast(Rn)
    out.trans = -np.einsum("nij,nj->ni", Rn, cn)
    out.points = scene.points + rng.normal(size=scene.points.shape) * point_frac * 3.0 / np.sqrt(3)
    return out


@dataclasses.dataclass
class RigDataset:
    """A rig problem with everything the mapper takes (``mapper.GlobalMapper.Solve``)."""
    scene: RigScene           # ground truth: poses, cam_from_rig, points and their observations
    view_graph: ViewGraph     # image level (image k = row k of the scene's image table)
    matches: dict             # make_pair_matches of scene.images_scene()
    features: dict            # {image id: [n,2] pixels}, image id k = image k
    image_pairs: list         # track_establishment.ImagePairMatches, every match an inlier


def make_rig_dataset(num_rigs: int, cameras_per_rig: int, frames_per_rig: int, num_points: int,
                     sensor_from_rig_translation_stddev: float = 0.1, sensor_from_rig_rotation_stddev: float = 5.0,
                     pixel_sigma: float = 0.0, seed: int = 1, rotation_noise_deg: float = 0.0, min_shared: int = 10,
                     model: int = SIMPLE_PINHOLE, focal: float = 1000.0, image_size: int = 1000,
                     world_scale: float = 0.1) -> RigDataset:
    """Rigs in the shape of ``colmap::SynthesizeDataset``: ``num_rigs`` rigs of ``cameras_per_rig`` cameras, each with
    ``frames_per_rig`` frames (frame f belongs to rig f // frames_per_rig; rig r owns sensors r * cameras_per_rig ...,
    the first its reference sensor with the identity cam_from_rig).  The other sensors are turned by a normal rotation
    vector of ``sensor_from_rig_rotation_stddev`` degrees per axis and shifted by a normal translation of
    ``sensor_from_rig_translation_stddev`` per axis.  Every sensor has its own intrinsics block and is known.  Frames sit on
    a shell r in [8, 12] * ``world_scale`` looking at a ball of radius 3 * ``world_scale``; every image that sees a point
    observes it, with ``pixel_sigma`` pixels of noise.  The default ``world_scale`` puts the points about one unit from
    the frames: global positioning fixes its gauge by holding one observation's scale and the rig scale at 1
    (global_positioning.cc:484-497), so known cam_from_rig translations agree with its solution only in a world of
    about that size.  The view graph is ``view_graph_from_scene`` of ``images_scene()`` (pairs sharing >= ``min_shared``
    points, ``rotation_noise_deg`` of rotation noise), the matches ``make_pair_matches`` without outliers."""
    rng = np.random.default_rng([seed, 101])
    R_, C_, F_ = int(num_rigs), int(cameras_per_rig), int(frames_per_rig)
    F, S = R_ * F_, R_ * C_
    Rf, tf = make_cameras(F, seed=seed, jitter_deg=5.0)
    tf = tf * world_scale
    w = rng.normal(size=(S, 3)) * np.radians(sensor_from_rig_rotation_stddev)
    ts = rng.normal(size=(S, 3)) * sensor_from_rig_translation_stddev
    ref = np.arange(R_) * C_
    w[ref], ts[ref] = 0.0, 0.0
    _, intr_model, intr_params = make_intrinsics(S, model, focal, image_size, S)
    frame_rig = (np.arange(F) // F_).astype(np.int32)
    image_frame = np.repeat(np.arange(F), C_).astype(np.int32)
    image_sensor = (frame_rig[image_frame] * C_ + np.tile(np.arange(C_), F)).astype(np.int32)
    scene = RigScene(geo.rotmat_to_quat_xyzw_fast(Rf), tf, np.zeros((0, 3)), np.zeros(1, np.int64), np.zeros(0, np.int32),
                     np.zeros(0, np.uint16), np.zeros((0, 2)), geo.rotmat_to_quat_xyzw_fast(geo.so3_exp(w)), ts,
                     np.arange(S, dtype=np.int32), intr_model, intr_params, image_frame, image_sensor, frame_rig,
                     (np.arange(S) // C_).astype(np.int32), ref.astype(np.int32), np.ones(S, bool))
    Ri, ti = scene.image_poses()
    d = rng.normal(size=(num_points, 3))
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    points = d * 3.0 * world_scale * rng.uniform(0, 1, size=(num_points, 1)) ** (1 / 3)
    Xc = np.einsum("nij,pj->pni", Ri, points) + ti[None]                   # [P, I, 3]
    lim = 0.5 * image_size / focal * 1.2
    with np.errstate(divide="ignore", invalid="ignore"):
        vis = (Xc[..., 2] > 0.5 * world_scale) & (np.abs(Xc[..., 0] / Xc[..., 2]) < lim) & (np.abs(Xc[..., 1] / Xc[..., 2]) < lim)
    p_idx, img = np.nonzero(vis)                                            # by point, then by image
    xy = np.empty((len(img), 2))
    for s in range(S):
        m = image_sensor[img] == s
        xy[m] = project(int(intr_model[s]), intr_params[s], Xc[p_idx[m], img[m]])
    if pixel_sigma > 0:
        xy += rng.normal(size=xy.shape) * pixel_sigma
    scene.points = points
    scene.pt_obs_begin = np.concatenate([[0], np.cumsum(vis.sum(1))]).astype(np.int64)
    scene.obs_frame, scene.obs_sensor = image_frame[img], image_sensor[img].astype(np.uint16)
    scene.obs_xy = xy
    images = scene.images_scene()
    vg = view_graph_from_scene(images, min_shared=min_shared, seed=seed, noise_deg=rotation_noise_deg)
    matches = make_pair_matches(images, seed=seed, outlier_frac=0.0)
    features, _, pairs = pairs_from_match_arrays(matches)
    for p in pairs:
        p.inliers = np.arange(len(p.matches))
    return RigDataset(scene, vg, matches, features, pairs)


def bearings_from_scene(scene: Scene) -> np.ndarray:
    """Unit bearing of each observation in the camera frame -- what the
    reference keeps in ``Image::features_undist`` (glomap/scene/image.h:31,
    processors/image_undistorter.cc).  Exact inverse for the pinhole models;
    radial models are inverted on the radius (``undistort_radius_scale``)."""
    out = np.empty((scene.N, 3))
    ci = scene.cam_intr[scene.obs_cam]
    for k in range(len(scene.intr_model)):
        mk = ci == k
        if not mk.any():
            continue
        out[mk] = bearings_from_pixels(int(scene.intr_model[k]), scene.intr_params[k], scene.obs_xy[mk])
    return out


UNDISTORT_MAX_ITERS = 100


def radial_fold_s(k1: float, k2: float) -> float:
    """The smallest positive s = r^2 where d/dr [r (1 + k1 r^2 + k2 r^4)] = 1 + 3 k1 s + 5 k2 s^2 reaches 0, or -1 when
    there is none."""
    if k2 == 0.0:
        return -1.0 / (3.0 * k1) if k1 < 0.0 else -1.0
    disc = 9.0 * k1 * k1 - 20.0 * k2
    if disc < 0.0:
        return -1.0
    q = -0.5 * (3.0 * k1 + np.copysign(np.sqrt(disc), k1))      # roots q / (5 k2) and 1 / q
    a, b = q / (5.0 * k2), 1.0 / q
    s = a if a > 0.0 else -1.0
    if b > 0.0 and (s < 0.0 or b < s):
        s = b
    return s


def undistort_radius_scale(k1: float, k2: float, rd: np.ndarray) -> np.ndarray:
    """r / rd for the r in [0, r_fold] with r (1 + k1 r^2 + k2 r^4) = rd (1 where rd = 0): Newton from r = rd inside a
    bracket kept by the sign of the residual, a bisection where a step leaves it, until a step no longer moves r or
    after ``UNDISTORT_MAX_ITERS``.  g(r) = r d(r^2) increases up to its fold (``radial_fold_s``); without one the root is
    below 2.25 rd, as d(r^2) > 4/9 there.  Past the fold there is no inverse and the result (r_fold at most) is not
    meant to be used.  The same steps as ``undistort_radius_scale`` in csrc/processor_kernels.cuh."""
    rd = np.asarray(rd, np.float64)
    s_fold = radial_fold_s(float(k1), float(k2))
    lo = np.zeros_like(rd)
    hi = np.full_like(rd, np.sqrt(s_fold)) if s_fold > 0.0 else 2.25 * rd
    r = np.minimum(rd, hi)
    act = rd > 0.0
    for _ in range(UNDISTORT_MAX_ITERS):
        if not act.any():
            break
        ra = r[act]
        s = ra * ra
        f = ra * (1.0 + s * (k1 + k2 * s)) - rd[act]
        la, ha = lo[act], hi[act]
        la = np.where(f < 0.0, ra, la)
        ha = np.where(f < 0.0, ha, ra)
        df = 1.0 + s * (3.0 * k1 + 5.0 * k2 * s)
        with np.errstate(divide="ignore", invalid="ignore"):
            rn = ra - f / df
        rn = np.where((rn >= la) & (rn <= ha), rn, 0.5 * (la + ha))
        lo[act], hi[act] = la, ha
        moved = rn != ra
        r[act] = rn
        act[act] = moved
    with np.errstate(divide="ignore", invalid="ignore"):
        return np.where(rd > 0.0, r / rd, 1.0)


def bearings_from_pixels(m: int, p: np.ndarray, xy: np.ndarray) -> np.ndarray:
    """``CamFromImg(xy).homogeneous().normalized()`` of [n,2] pixels of one camera (model ``m``, parameters ``p``)."""
    if m == SIMPLE_PINHOLE:
        u, v = (xy[:, 0] - p[1]) / p[0], (xy[:, 1] - p[2]) / p[0]
    elif m == PINHOLE:
        u, v = (xy[:, 0] - p[2]) / p[0], (xy[:, 1] - p[3]) / p[1]
    else:
        ud, vd = (xy[:, 0] - p[1]) / p[0], (xy[:, 1] - p[2]) / p[0]
        sc = undistort_radius_scale(p[3], p[4] if m == RADIAL else 0.0, np.sqrt(ud * ud + vd * vd))
        u, v = ud * sc, vd * sc
    b = np.stack([u, v, np.ones_like(u)], 1)
    return b / np.linalg.norm(b, axis=1, keepdims=True)


# ---------------------------------------------------------------------------
# View graphs for rotation averaging
# ---------------------------------------------------------------------------
@dataclasses.dataclass
class ViewGraph:
    """Flat view graph: edge e relates images (i, j) with R_rel = R_j R_i^T
    (``cam2_from_cam1`` of the reference, glomap/scene/image_pair.h)."""
    n_images: int
    ei: np.ndarray      # [E] int32 image index 1
    ej: np.ndarray      # [E] int32 image index 2
    R_rel: np.ndarray   # [E,3,3]
    weight: np.ndarray  # [E]
    R_gt: np.ndarray    # [n,3,3] ground-truth cam_from_world rotations

    @property
    def E(self):
        return len(self.ei)


def _noisy_relative(R_gt, ei, ej, rng, noise_deg, outlier_ratio):
    R_rel = R_gt[ej] @ np.swapaxes(R_gt[ei], -1, -2)
    E = len(ei)
    if noise_deg > 0:
        w = rng.normal(size=(E, 3)) * np.radians(noise_deg) / np.sqrt(3)
        R_rel = geo.so3_exp(w) @ R_rel
    if outlier_ratio > 0:
        out = rng.uniform(size=E) < outlier_ratio
        w = rng.normal(size=(int(out.sum()), 3))
        w /= np.linalg.norm(w, axis=1, keepdims=True)
        w *= rng.uniform(0, np.pi, size=(len(w), 1))
        R_rel[out] = geo.so3_exp(w)
    return R_rel


def make_ring_view_graph(n: int = 100, k: int = 5, seed: int = 1, noise_deg: float = 0.0,
                         outlier_ratio: float = 0.0) -> ViewGraph:
    """Config 1: n cameras on a ring of radius 10 looking at the centre,
    edges (i, i+d mod n) for d = 1..k."""
    rng = np.random.default_rng(seed)
    ang = 2 * np.pi * np.arange(n) / n
    centers = np.stack([10 * np.sin(ang), np.zeros(n), 10 * np.cos(ang)], 1)
    R_gt = _look_at_rotations(centers, rng, 0.0)
    ei = np.repeat(np.arange(n), k)
    ej = (ei + np.tile(np.arange(1, k + 1), n)) % n
    R_rel = _noisy_relative(R_gt, ei, ej, rng, noise_deg, outlier_ratio)
    return ViewGraph(n, ei.astype(np.int32), ej.astype(np.int32), R_rel, np.ones(len(ei)), R_gt)


def make_random_view_graph(n: int, avg_degree: float, seed: int = 1, noise_deg: float = 0.0,
                           outlier_ratio: float = 0.0) -> ViewGraph:
    """Random rotations, a spanning path for connectivity plus random edges."""
    rng = np.random.default_rng(seed)
    w = rng.normal(size=(n, 3))
    w /= np.linalg.norm(w, axis=1, keepdims=True)
    w *= rng.uniform(0, np.pi, size=(n, 1))
    R_gt = geo.so3_exp(w)
    perm = rng.permutation(n)
    pairs = {(min(a, b), max(a, b)) for a, b in zip(perm[:-1], perm[1:])}
    target = int(n * avg_degree / 2)
    while len(pairs) < target:
        a = rng.integers(0, n, size=target)
        b = rng.integers(0, n, size=target)
        for x, y in zip(a, b):
            if x != y:
                pairs.add((min(x, y), max(x, y)))
            if len(pairs) >= target:
                break
    pr = np.array(sorted(pairs), dtype=np.int64)
    ei, ej = pr[:, 0], pr[:, 1]
    R_rel = _noisy_relative(R_gt, ei, ej, rng, noise_deg, outlier_ratio)
    return ViewGraph(n, ei.astype(np.int32), ej.astype(np.int32), R_rel, np.ones(len(ei)), R_gt)


def make_lattice_view_graph(n: int = 100_000, neighbours: int = 50, seed: int = 1, noise_deg: float = 2.0,
                            outlier_ratio: float = 0.05) -> ViewGraph:
    """Config 5: cameras on a 2-D lattice, each linked to its ``neighbours``
    nearest lattice neighbours (half of them stored, i<j)."""
    rng = np.random.default_rng(seed)
    side = int(np.ceil(np.sqrt(n)))
    gx, gy = np.divmod(np.arange(n), side)
    w = rng.normal(size=(n, 3)) * 0.5
    R_gt = geo.so3_exp(w)
    rad = 1
    while (2 * rad + 1) ** 2 - 1 < neighbours:
        rad += 1
    offs = [(dx, dy) for dx in range(-rad, rad + 1) for dy in range(-rad, rad + 1) if (dx, dy) > (0, 0)]
    offs.sort(key=lambda o: o[0] * o[0] + o[1] * o[1])
    offs = offs[: neighbours // 2]
    ei_l, ej_l = [], []
    for dx, dy in offs:
        nx, ny = gx + dx, gy + dy
        j = nx * side + ny
        ok = (nx >= 0) & (nx < side) & (ny >= 0) & (ny < side) & (j < n)
        ei_l.append(np.arange(n)[ok])
        ej_l.append(j[ok])
    ei = np.concatenate(ei_l)
    ej = np.concatenate(ej_l)
    R_rel = _noisy_relative(R_gt, ei, ej, rng, noise_deg, outlier_ratio)
    return ViewGraph(n, ei.astype(np.int32), ej.astype(np.int32), R_rel, np.ones(len(ei)), R_gt)


def view_graph_from_scene(scene: Scene, min_shared: int = 30, seed: int = 3, noise_deg: float = 0.0,
                          outlier_ratio: float = 0.0) -> ViewGraph:
    """Camera pairs sharing >= ``min_shared`` points, with relative rotations
    from the scene's rotations (config 2's view graph)."""
    import scipy.sparse as sp
    rng = np.random.default_rng(seed)
    pt_of_obs = np.repeat(np.arange(scene.P), np.diff(scene.pt_obs_begin))
    V = sp.csr_matrix((np.ones(scene.N, dtype=np.int32), (scene.obs_cam, pt_of_obs)), shape=(scene.C, scene.P))
    cov = sp.triu(V @ V.T, k=1).tocoo()
    keep = cov.data >= min_shared
    ei, ej = cov.row[keep], cov.col[keep]
    R_gt = geo.quat_xyzw_to_rotmat(scene.quat)
    R_rel = _noisy_relative(R_gt, ei, ej, rng, noise_deg, outlier_ratio)
    return ViewGraph(scene.C, ei.astype(np.int32), ej.astype(np.int32), R_rel, cov.data[keep].astype(np.float64), R_gt)


# ---------------------------------------------------------------------------
# Text formats of `glomap rotation_averager` (docs/rotation_averager.md:43-69)
# ---------------------------------------------------------------------------
def write_relpose_file(path: str, vg: ViewGraph, names=None) -> None:
    """IMAGE_NAME_1 IMAGE_NAME_2 QW QX QY QZ TX TY TZ (glomap/io/pose_io.cc:36-75)."""
    names = names or [f"img{i:04d}" for i in range(vg.n_images)]
    q = geo.rotmat_to_quat_xyzw_fast(vg.R_rel)
    with open(path, "w") as f:
        for e in range(vg.E):
            f.write(f"{names[vg.ei[e]]} {names[vg.ej[e]]} {q[e,3]:.17g} {q[e,0]:.17g} {q[e,1]:.17g} {q[e,2]:.17g} 1 0 0\n")


def read_relpose_file(path: str) -> tuple[ViewGraph, list[str]]:
    """Parser with the reference's id assignment: images numbered in order of
    first appearance (glomap/io/pose_io.cc:46-59)."""
    names, idx, ei, ej, qs = [], {}, [], [], []
    with open(path) as f:
        for line in f:
            tok = line.rstrip("\n").split(" ")
            if len(tok) < 9:
                continue
            for nm in tok[:2]:
                if nm not in idx:
                    idx[nm] = len(names)
                    names.append(nm)
            ei.append(idx[tok[0]])
            ej.append(idx[tok[1]])
            qw, qx, qy, qz = (float(x) for x in tok[2:6])
            qs.append([qx, qy, qz, qw])
    R_rel = geo.quat_xyzw_to_rotmat(np.array(qs))
    n = len(names)
    vg = ViewGraph(n, np.array(ei, np.int32), np.array(ej, np.int32), R_rel, np.ones(len(ei)), np.tile(np.eye(3), (n, 1, 1)))
    return vg, names


def write_global_rotation_file(path: str, names, R: np.ndarray) -> None:
    """IMAGE_NAME QW QX QY QZ, default ostream precision (pose_io.cc:182-200)."""
    q = geo.rotmat_to_quat_xyzw_fast(R)
    with open(path, "w") as f:
        for i, nm in enumerate(names):
            f.write(f"{nm} {q[i,3]:.6g} {q[i,0]:.6g} {q[i,1]:.6g} {q[i,2]:.6g}\n")


# ---------------------------------------------------------------------------
# Flat binary problem file (glomap_b200/host/b200sfm_cli.cc)
# ---------------------------------------------------------------------------
def write_flat_problem(path: str, scene: Scene, bearings: np.ndarray | None = None) -> None:
    """int64 {C,P,N,K}; int64 pt_obs_begin[P+1]; int32 obs_cam[N]; f64 obs_xy[2N]; f64 bearings[3N];
    int32 cam_intr[C]; int32 intr_model[K]; f64 intr[K*12]; f64 quat[4C]; f64 trans[3C]; f64 points[3P]."""
    b = bearings_from_scene(scene) if bearings is None else bearings
    with open(path, "wb") as f:
        np.array([scene.C, scene.P, scene.N, len(scene.intr_model)], np.int64).tofile(f)
        for arr, dt in ((scene.pt_obs_begin, np.int64), (scene.obs_cam, np.int32), (scene.obs_xy, np.float64),
                        (b, np.float64), (scene.cam_intr, np.int32), (scene.intr_model, np.int32),
                        (scene.intr_params, np.float64), (scene.quat, np.float64), (scene.trans, np.float64),
                        (scene.points, np.float64)):
            np.ascontiguousarray(arr, dtype=dt).tofile(f)


def read_flat_problem(path: str) -> Scene:
    with open(path, "rb") as f:
        C, P, N, K = (int(x) for x in np.fromfile(f, np.int64, 4))
        ptb = np.fromfile(f, np.int64, P + 1)
        cam = np.fromfile(f, np.int32, N)
        xy = np.fromfile(f, np.float64, 2 * N).reshape(N, 2)
        np.fromfile(f, np.float64, 3 * N)
        ci = np.fromfile(f, np.int32, C)
        im = np.fromfile(f, np.int32, K)
        intr = np.fromfile(f, np.float64, K * INTR_STRIDE).reshape(K, INTR_STRIDE)
        quat = np.fromfile(f, np.float64, 4 * C).reshape(C, 4)
        trans = np.fromfile(f, np.float64, 3 * C).reshape(C, 3)
        pts = np.fromfile(f, np.float64, 3 * P).reshape(P, 3)
    return Scene(quat, trans, pts, ptb, cam, xy, ci, im, intr)


# ---------------------------------------------------------------------------
# Image pairs with matches (input of ImagePairsInlierCount)
# ---------------------------------------------------------------------------
def _pinhole_K(model: int, p: np.ndarray) -> np.ndarray:
    fx, fy, cx, cy = (p[0], p[1], p[2], p[3]) if model == PINHOLE else (p[0], p[0], p[1], p[2])
    return np.array([[fx, 0.0, cx], [0.0, fy, cy], [0.0, 0.0, 1.0]])


def _fit_homography(x1: np.ndarray, x2: np.ndarray) -> np.ndarray:
    """Least-squares homography x2 ~ H x1 (normalised DLT)."""
    def norm(x):
        c = x.mean(0)
        s = np.sqrt(2.0) / max(np.linalg.norm(x - c, axis=1).mean(), 1e-12)
        return np.array([[s, 0, -s * c[0]], [0, s, -s * c[1]], [0, 0, 1.0]])
    T1, T2 = norm(x1), norm(x2)
    a = x1 @ T1[:2, :2].T + T1[:2, 2]
    b = x2 @ T2[:2, :2].T + T2[:2, 2]
    z, o = np.zeros(len(a)), np.ones(len(a))
    A = np.concatenate([np.stack([a[:, 0], a[:, 1], o, z, z, z, -b[:, 0] * a[:, 0], -b[:, 0] * a[:, 1], -b[:, 0]], 1),
                        np.stack([z, z, z, a[:, 0], a[:, 1], o, -b[:, 1] * a[:, 0], -b[:, 1] * a[:, 1], -b[:, 1]], 1)])
    Hn = np.linalg.svd(A)[2][-1].reshape(3, 3)
    H = np.linalg.inv(T2) @ Hn @ T1
    return H / H[2, 2]


def make_pair_matches(scene: Scene, seed: int = 1, outlier_frac: float = 0.2, config_weights=(0.8, 0.15, 0.05)) -> dict:
    """Flat image-pair match set from the tracks of ``scene``: feature f of image i is the f-th observation of camera i
    (in observation order); every pair of observations inside a track is a match of the pair (i < j) of their cameras;
    ``outlier_frac`` of the final matches are random feature pairs of the same image pairs.  Each pair is CALIBRATED,
    UNCALIBRATED or PLANAR with the probabilities ``config_weights`` and carries the true cam2_from_cam1 (unit
    translation), the F of the
    pinhole part of the two cameras and, for PLANAR pairs, the least-squares homography of its true matches (the infinite
    homography K2 R K1^-1 when it has fewer than 4).  Arrays (the layout of
    b200sfm_image_pairs_inlier_count): feature_begin [C+1], features [nf,2], image_intr [C], intr_model, intr_params,
    img1/img2/config [E], quat [E,4], trans [E,3], F/H [E,9], match_begin [E+1], matches [M,2] int32, is_true [M]."""
    rng = np.random.default_rng([seed, 77])
    C = scene.C
    counts = np.bincount(scene.obs_cam, minlength=C)
    feature_begin = np.concatenate([[0], np.cumsum(counts)]).astype(np.int64)
    order = np.argsort(scene.obs_cam, kind="stable")
    feat_of_obs = np.empty(scene.N, np.int64)
    feat_of_obs[order] = np.arange(scene.N) - feature_begin[scene.obs_cam[order]]
    lens = np.diff(scene.pt_obs_begin)
    us, vs = [], []
    for L in np.unique(lens[lens >= 2]):
        starts = scene.pt_obs_begin[:-1][lens == L]
        a, b = np.triu_indices(int(L), 1)
        us.append((starts[:, None] + a[None, :]).ravel())
        vs.append((starts[:, None] + b[None, :]).ravel())
    u, v = np.concatenate(us), np.concatenate(vs)
    ci, cj = scene.obs_cam[u].astype(np.int64), scene.obs_cam[v].astype(np.int64)
    fu, fv = feat_of_obs[u], feat_of_obs[v]
    swap = ci > cj
    ci, cj, fu, fv = np.where(swap, cj, ci), np.where(swap, ci, cj), np.where(swap, fv, fu), np.where(swap, fu, fv)
    del u, v, swap
    n_out = int(round(len(ci) * outlier_frac / (1.0 - outlier_frac)))
    src = rng.integers(0, len(ci), n_out)
    oi, oj = ci[src], cj[src]
    of1 = (rng.random(n_out) * counts[oi]).astype(np.int64)
    of2 = (rng.random(n_out) * counts[oj]).astype(np.int64)
    is_true = np.concatenate([np.ones(len(ci), bool), np.zeros(n_out, bool)])
    key = np.concatenate([ci * C + cj, oi * C + oj])
    f1, f2 = np.concatenate([fu, of1]), np.concatenate([fv, of2])
    del ci, cj, fu, fv, oi, oj, of1, of2, src
    perm = np.lexsort((rng.random(len(key)), key))             # by pair; true and outlier matches interleaved
    key, is_true = key[perm], is_true[perm]
    matches = np.stack([f1[perm], f2[perm]], 1).astype(np.int32)
    del f1, f2, perm
    heads = np.concatenate([[0], np.nonzero(np.diff(key))[0] + 1]) if len(key) else np.zeros(0, np.int64)
    match_begin = np.concatenate([heads, [len(key)]]).astype(np.int64)
    img1, img2 = (key[heads] // C).astype(np.int32), (key[heads] % C).astype(np.int32)
    E = len(heads)
    config = rng.choice(np.array([2, 3, 4], np.int32), size=E, p=np.asarray(config_weights, float) / np.sum(config_weights))
    R = geo.quat_xyzw_to_rotmat(scene.quat)
    R_rel = R[img2] @ np.swapaxes(R[img1], -1, -2)
    t_rel = scene.trans[img2] - np.einsum("nij,nj->ni", R_rel, scene.trans[img1])
    t_rel /= np.linalg.norm(t_rel, axis=1, keepdims=True)     # unit baseline, as relative pose estimation returns it
    Kinv = np.array([np.linalg.inv(_pinhole_K(int(m), p)) for m, p in zip(scene.intr_model, scene.intr_params)])
    Kb = np.array([_pinhole_K(int(m), p) for m, p in zip(scene.intr_model, scene.intr_params)])
    K1i, K2i = Kinv[scene.cam_intr[img1]], Kinv[scene.cam_intr[img2]]
    tx = np.zeros((E, 3, 3))
    tx[:, 0, 1], tx[:, 0, 2], tx[:, 1, 2] = -t_rel[:, 2], t_rel[:, 1], -t_rel[:, 0]
    tx[:, 1, 0], tx[:, 2, 0], tx[:, 2, 1] = t_rel[:, 2], -t_rel[:, 1], t_rel[:, 0]
    F = np.swapaxes(K2i, -1, -2) @ tx @ R_rel @ K1i
    F /= np.linalg.norm(F.reshape(E, 9), axis=1)[:, None, None]
    H = Kb[scene.cam_intr[img2]] @ R_rel @ K1i
    feats = scene.obs_xy[order]
    for e in np.nonzero(config == 4)[0]:     # PLANAR: the DLT homography of the pair's true matches, where there are 4
        m = matches[match_begin[e]:match_begin[e + 1]][is_true[match_begin[e]:match_begin[e + 1]]]
        if len(m) >= 4:
            H[e] = _fit_homography(feats[feature_begin[img1[e]] + m[:, 0]], feats[feature_begin[img2[e]] + m[:, 1]])
    return dict(feature_begin=feature_begin, features=np.ascontiguousarray(scene.obs_xy[order]),
                image_intr=scene.cam_intr.astype(np.int32), intr_model=scene.intr_model.astype(np.int32),
                intr_params=scene.intr_params, img1=img1, img2=img2, config=config.astype(np.int32),
                quat=geo.rotmat_to_quat_xyzw_fast(R_rel), trans=t_rel, F=F.reshape(E, 9), H=H.reshape(E, 9),
                match_begin=match_begin, matches=matches, is_true=is_true)


def pairs_from_match_arrays(d: dict):
    """(features, cameras, pairs) of ``make_pair_matches`` arrays for the object-level API (image_pair_inliers.py): image
    ids are the camera indices, every image has its own camera object, pairs carry no inliers."""
    from .image_pair_inliers import Camera
    from .track_establishment import ImagePairMatches
    C = len(d["image_intr"])
    fb = d["feature_begin"]
    features = {i: d["features"][fb[i]:fb[i + 1]] for i in range(C)}
    cameras = {i: Camera(int(d["intr_model"][d["image_intr"][i]]), d["intr_params"][d["image_intr"][i]]) for i in range(C)}
    mb = d["match_begin"]
    pairs = [ImagePairMatches(int(d["img1"][e]), int(d["img2"][e]), d["matches"][mb[e]:mb[e + 1]], np.zeros(0, np.int64),
                              config=int(d["config"][e]), quat_xyzw=d["quat"][e], trans=d["trans"][e],
                              F=d["F"][e].reshape(3, 3), H=d["H"][e].reshape(3, 3)) for e in range(len(d["img1"]))]
    return features, cameras, pairs


# ---------------------------------------------------------------------------
# Fundamental matrices of camera pairs (input of ViewGraphCalibrator)
# ---------------------------------------------------------------------------
def make_vgc_pairs(scene: Scene, pairs, seed: int = 1, f_noise: float = 0.0, outlier_frac: float = 0.0,
                   F_sigma: float = 0.0) -> dict:
    """F of the image pairs ``pairs`` ([E, 2] image indices) of ``scene``, without matches: F = K2^-T [t]x R K1^-1 of the
    true poses and the pinhole part of the true intrinsics (the camera of image i is intrinsics block cam_intr[i]),
    normalised to unit Frobenius norm.  ``F_sigma`` multiplies every entry by 1 + N(0, F_sigma^2); ``outlier_frac`` of the
    pairs get a random unit-norm F instead (``is_outlier``).  ``focal_init`` [K] is Camera::Focal() of each block times
    (1 + U(-f_noise, f_noise)).  Arrays: img1, img2, cam1, cam2 [E] int32, F [E, 9], principal_point [K, 2], focal_true,
    focal_init [K], is_outlier [E]."""
    rng = np.random.default_rng([seed, 91])
    pr = np.asarray(pairs, np.int64).reshape(-1, 2)
    img1, img2 = pr[:, 0], pr[:, 1]
    E = len(pr)
    R = geo.quat_xyzw_to_rotmat(scene.quat)
    R_rel = R[img2] @ np.swapaxes(R[img1], -1, -2)
    t_rel = scene.trans[img2] - np.einsum("nij,nj->ni", R_rel, scene.trans[img1])
    t_rel /= np.linalg.norm(t_rel, axis=1, keepdims=True)
    Kinv = np.array([np.linalg.inv(_pinhole_K(int(m), p)) for m, p in zip(scene.intr_model, scene.intr_params)])
    cam1, cam2 = scene.cam_intr[img1].astype(np.int32), scene.cam_intr[img2].astype(np.int32)
    tx = np.zeros((E, 3, 3))
    tx[:, 0, 1], tx[:, 0, 2], tx[:, 1, 2] = -t_rel[:, 2], t_rel[:, 1], -t_rel[:, 0]
    tx[:, 1, 0], tx[:, 2, 0], tx[:, 2, 1] = t_rel[:, 2], -t_rel[:, 1], t_rel[:, 0]
    F = (np.swapaxes(Kinv[cam2], -1, -2) @ tx @ R_rel @ Kinv[cam1]).reshape(E, 9)
    F /= np.linalg.norm(F, axis=1, keepdims=True)
    if F_sigma > 0:
        F *= 1.0 + rng.normal(scale=F_sigma, size=F.shape)
    is_outlier = rng.random(E) < outlier_frac
    n_out = int(is_outlier.sum())
    Fo = rng.normal(size=(n_out, 9))
    F[is_outlier] = Fo / np.linalg.norm(Fo, axis=1, keepdims=True)
    p = scene.intr_params
    pinhole = scene.intr_model == PINHOLE
    focal_true = np.where(pinhole, (p[:, 0] + p[:, 1]) / 2.0, p[:, 0])
    principal_point = np.where(pinhole[:, None], p[:, 2:4], p[:, 1:3])
    focal_init = focal_true * (1.0 + rng.uniform(-f_noise, f_noise, size=len(focal_true)))
    return dict(img1=img1.astype(np.int32), img2=img2.astype(np.int32), cam1=cam1, cam2=cam2, F=np.ascontiguousarray(F),
                principal_point=np.ascontiguousarray(principal_point), focal_true=focal_true, focal_init=focal_init,
                is_outlier=is_outlier)


def make_calibration_pairs(scene: Scene, pairs, seed: int = 1, uncalibrated_frac: float = 0.3, outlier_frac: float = 0.0):
    """Image pairs for stages 0 and 1 of the mapper (``view_graph_manipulation`` / ``view_graph_calibration``) over the
    image pairs ``pairs`` ([E, 2] image indices = image ids) of ``scene``: ``track_establishment.ImagePairMatches``
    without matches, with the true cam2_from_cam1 (unit translation) and the F of ``make_vgc_pairs``.  A pair is
    UNCALIBRATED with probability ``uncalibrated_frac``, else CALIBRATED.  ``outlier_frac`` of the pairs are CALIBRATED
    outliers whose F is that of the true pose with both focal lengths three times too large: its Fetzer residuals at the
    true focals are -8, far above ViewGraphCalibrator's threshold (a random F often stays under it).  Stage 0 recomputes
    the F of the UNCALIBRATED pairs it promotes, so no outlier is UNCALIBRATED.  Returns (pairs, is_outlier [E])."""
    from .track_establishment import ImagePairMatches
    d = make_vgc_pairs(scene, pairs, seed=seed)
    rng = np.random.default_rng([seed, 93])
    img1, img2 = d["img1"].astype(np.int64), d["img2"].astype(np.int64)
    R = geo.quat_xyzw_to_rotmat(scene.quat)
    R_rel = R[img2] @ np.swapaxes(R[img1], -1, -2)
    t_rel = scene.trans[img2] - np.einsum("nij,nj->ni", R_rel, scene.trans[img1])
    t_rel /= np.linalg.norm(t_rel, axis=1, keepdims=True)
    q_rel = geo.rotmat_to_quat_xyzw_fast(R_rel)
    is_outlier = rng.random(len(img1)) < outlier_frac
    scaled = scene.intr_params.copy()
    scaled[:, 0] *= 3.0
    scaled[scene.intr_model == PINHOLE, 1] *= 3.0
    Kinv = np.array([np.linalg.inv(_pinhole_K(int(m), p)) for m, p in zip(scene.intr_model, scaled)])
    for e in np.flatnonzero(is_outlier):
        tx = np.array([[0.0, -t_rel[e, 2], t_rel[e, 1]], [t_rel[e, 2], 0.0, -t_rel[e, 0]], [-t_rel[e, 1], t_rel[e, 0], 0.0]])
        Fo = Kinv[scene.cam_intr[img2[e]]].T @ tx @ R_rel[e] @ Kinv[scene.cam_intr[img1[e]]]
        d["F"][e] = (Fo / np.linalg.norm(Fo)).ravel()
    uncal = (rng.random(len(img1)) < uncalibrated_frac) & ~is_outlier
    out = [ImagePairMatches(int(img1[e]), int(img2[e]), np.zeros((0, 2), np.int32), np.zeros(0, np.int64),
                            config=3 if uncal[e] else 2, quat_xyzw=q_rel[e].copy(), trans=t_rel[e].copy(),
                            F=d["F"][e].reshape(3, 3).copy()) for e in range(len(img1))]
    return out, is_outlier


# ---------------------------------------------------------------------------
# Covisibility clusters (input of PruneWeaklyConnectedImages)
# ---------------------------------------------------------------------------
def make_cluster_tracks(group_sizes, tracks_per_window: int = 40, bridges=(), seed: int = 1, shuffle: bool = True) -> dict:
    """Frame groups with dense internal tracks plus bridge tracks of set covisibility counts.

    Group g of n_g >= 4 frames gets ``tracks_per_window`` = K tracks over every window of 3 consecutive frames of the
    group, so its adjacent frame pairs are seen together 2K times (K at the two ends) and the pairs two apart K times.
    With fewer than 3 bridges per group the median edge weight is K and the MAD 0, so the strong-cluster threshold is
    thr = max(K, 20): the interior adjacent pairs are strong edges and the end frames join through their two weaker ones,
    so each group is one cluster.  A bridge (a, b, c) (global frame indices before shuffling, c >= 2) adds tracks
    [a, a, b] (2 counts of (a, b) each; one [a, a, a, b] when c is odd) and no other pair, so two groups merge when
    c > thr, or when two bridges between them both have 0.75 thr <= c.

    ``shuffle`` relabels the frames with a random permutation and shuffles the tracks and the observations inside each
    track.  Returns dict(track_begin [T+1] int64, obs_frame [N] int32, num_frames, group [F] int32 (group of every frame
    after relabelling), threshold = max(K, 20))."""
    rng = np.random.default_rng([seed, 97])
    sizes = [int(n) for n in group_sizes]
    if min(sizes) < 4:
        raise ValueError("groups need >= 4 frames")
    F = sum(sizes)
    start = np.concatenate([[0], np.cumsum(sizes)])
    tracks = []
    for g, n in enumerate(sizes):
        for i in range(n - 2):
            tracks += [[start[g] + i, start[g] + i + 1, start[g] + i + 2]] * tracks_per_window
    for a, b, c in bridges:
        c = int(c)
        if c < 2:
            raise ValueError("a bridge count must be >= 2")
        if c % 2:
            tracks.append([a, a, a, b])
            c -= 3
        tracks += [[a, a, b]] * (c // 2)
    group = np.repeat(np.arange(len(sizes)), sizes).astype(np.int32)
    perm = rng.permutation(F) if shuffle else np.arange(F)
    tracks = [list(perm[np.asarray(t)]) for t in tracks]
    if shuffle:
        order = rng.permutation(len(tracks))
        tracks = [list(rng.permutation(tracks[k])) for k in order]
    new_group = np.empty(F, np.int32)
    new_group[perm] = group
    lens = np.array([len(t) for t in tracks], np.int64)
    track_begin = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
    obs_frame = np.concatenate([np.asarray(t, np.int64) for t in tracks]).astype(np.int32) if tracks else np.zeros(0, np.int32)
    return dict(track_begin=track_begin, obs_frame=obs_frame, num_frames=F, group=new_group,
                threshold=max(float(tracks_per_window), 20.0))


# ---------------------------------------------------------------------------
# Gravity priors (`glomap rotation_averager --gravity_path`, docs/rotation_averager.md)
# ---------------------------------------------------------------------------
def _random_axis_rotations(rng, k: int, angle_sigma: float) -> np.ndarray:
    """CreateRandomRotation (controllers/rotation_averager_test.cc:16-34): an axis uniform in (theta, phi) and a normal
    angle of standard deviation ``angle_sigma`` radians; returns rotation vectors [k,3]."""
    theta = rng.uniform(0, 2 * np.pi, size=k)
    phi = rng.uniform(0, np.pi, size=k)
    axis = np.stack([np.cos(theta) * np.sin(phi), np.sin(theta) * np.sin(phi), np.cos(phi)], 1)
    return axis * rng.normal(0, angle_sigma, size=(k, 1))


def make_gravity(R_gt: np.ndarray, noise_deg: float = 0.0, outlier_ratio: float = 0.0, seed: int = 1):
    """PrepareGravity (controllers/rotation_averager_test.cc:36-63): the gravity of frame f is R_gt[f] (0, 1, 0)
    (rig_from_world times the world's gravity), turned by a random rotation of ``noise_deg`` standard deviation; with
    probability ``outlier_ratio`` it is replaced by the unit rotation axis of a random rotation (1 rad standard
    deviation).  Returns (gravity [F,3], is_outlier [F])."""
    rng = np.random.default_rng(seed)
    R_gt = np.asarray(R_gt, dtype=np.float64)
    F = len(R_gt)
    g = R_gt[:, :, 1].copy()
    if noise_deg > 0:
        g = np.einsum("nij,nj->ni", geo.so3_exp(_random_axis_rotations(rng, F, np.radians(noise_deg))), g)
    out = rng.uniform(size=F) < outlier_ratio if outlier_ratio > 0 else np.zeros(F, bool)
    if out.any():
        w = _random_axis_rotations(rng, int(out.sum()), 1.0)
        g[out] = w / np.linalg.norm(w, axis=1, keepdims=True)
    return g, out


def make_frame_gravity(R_frames: np.ndarray, share: float = 1.0, noise_deg: float = 0.0, outlier_ratio: float = 0.0,
                       seed: int = 1) -> np.ndarray:
    """Gravity priors for the frames of a dataset (``GlobalMapper.Solve(..., gravity=...)``): ``make_gravity`` of the
    ground-truth rig_from_world (or cam_from_world) rotations ``R_frames`` [F,3,3], with each frame left without a prior
    (a NaN row) with probability 1 - ``share``.  Returns [F,3]."""
    g, _ = make_gravity(R_frames, noise_deg, outlier_ratio, seed)
    g[np.random.default_rng([seed, 13]).uniform(size=len(g)) >= share] = np.nan
    return g


def write_gravity_file(path: str, names, gravity: np.ndarray) -> None:
    """IMAGE_NAME GX GY GZ (glomap/io/pose_io.cc:139-180); rows of NaN (no prior) are not written."""
    with open(path, "w") as f:
        for nm, g in zip(names, np.asarray(gravity, dtype=np.float64)):
            if np.isfinite(g).all():
                f.write(f"{nm} {g[0]:.17g} {g[1]:.17g} {g[2]:.17g}\n")


def read_gravity_file(path: str, names) -> np.ndarray:
    """ReadGravity's parse: [len(names),3] with NaN rows for the images the file does not name; unknown names are
    ignored."""
    idx = {nm: i for i, nm in enumerate(names)}
    g = np.full((len(names), 3), np.nan)
    with open(path) as f:
        for line in f:
            tok = line.rstrip("\n").split(" ")
            if len(tok) >= 4 and tok[0] in idx:
                g[idx[tok[0]]] = [float(x) for x in tok[1:4]]
    return g


def write_weight_file(path: str, vg: ViewGraph, weight: np.ndarray, names=None) -> None:
    """IMAGE_NAME_1 IMAGE_NAME_2 WEIGHT (ReadRelWeight, glomap/io/pose_io.cc:91-135)."""
    names = names or [f"img{i:04d}" for i in range(vg.n_images)]
    with open(path, "w") as f:
        for e in range(vg.E):
            f.write(f"{names[vg.ei[e]]} {names[vg.ej[e]]} {float(weight[e]):.17g}\n")
