"""Flat problem  <->  COLMAP sparse model (``cameras.bin / images.bin / points3D.bin``) -- SURVEY.md 8(f) item 3.

The reference reads and writes its results through ``colmap::Reconstruction`` (glomap/io/colmap_io.cc:8-58,
glomap/io/colmap_converter.cc:22-133,137-213); COLMAP is not vendored, so the binary layout is restated here from the
public COLMAP sources (src/colmap/scene/reconstruction_io.cc, UPSTREAM-UNVERIFIED; little-endian, packed):

  cameras.bin   u64 n | n x { u32 camera_id, i32 model_id, u64 width, u64 height, f64 params[num_params(model)] }
  images.bin    u64 n | n x { u32 image_id, f64 qvec[4] (w x y z), f64 tvec[3] (cam_from_world), u32 camera_id,
                              char name[] NUL-terminated, u64 m, m x { f64 x, f64 y, u64 point3D_id (2^64-1 = none) } }
  points3D.bin  u64 n | n x { u64 point3D_id, f64 xyz[3], u8 rgb[3], f64 error, u64 L, L x { u32 image_id, u32 point2D_idx } }

Only trivial frames (one image per frame) are converted; models written by a rig-aware COLMAP additionally carry
``rigs.bin`` / ``frames.bin``, which are ignored on read and not written (COLMAP then creates trivial rigs).

``scene_from_model`` builds the SoA ``synthetic.Scene`` the C ABI consumes -- images, cameras and points in sorted-id
order (the order the C++ shim uses) -- plus a ``ModelIndex`` with everything needed to write the optimised state back;
``model_from_scene`` applies ConvertGlomapToColmap's rules: points with fewer than 2 supporting observations are
dropped (colmap_converter.cc:48,111), ``point3D_id`` is set on the observed features, ``error`` is the mean
reprojection error (Reconstruction::UpdatePoint3DErrors)."""
from __future__ import annotations

import dataclasses
import os
import struct

import numpy as np

from . import synthetic as S

NUM_PARAMS = {0: 3, 1: 4, 2: 4, 3: 5, 4: 8, 5: 8, 6: 12, 7: 5, 8: 4, 9: 5, 10: 12, 11: 16}
INVALID_POINT3D = np.uint64(2**64 - 1)
_P2D = np.dtype([("x", "<f8"), ("y", "<f8"), ("id", "<u8")])
_TRK = np.dtype([("image_id", "<u4"), ("point2D_idx", "<u4")])


@dataclasses.dataclass
class Camera:
    camera_id: int
    model_id: int
    width: int
    height: int
    params: np.ndarray


@dataclasses.dataclass
class Image:
    image_id: int
    qvec_wxyz: np.ndarray      # cam_from_world
    tvec: np.ndarray
    camera_id: int
    name: str
    xy: np.ndarray             # [m,2]
    point3D_ids: np.ndarray    # [m] uint64, INVALID_POINT3D = unobserved


@dataclasses.dataclass
class Point3D:
    point3D_id: int
    xyz: np.ndarray
    rgb: np.ndarray
    error: float
    image_ids: np.ndarray      # [L] uint32
    point2D_idxs: np.ndarray   # [L] uint32


# ---------------------------------------------------------------------------- raw model I/O
def read_cameras(path: str) -> dict[int, Camera]:
    out = {}
    with open(path, "rb") as f:
        (n,) = struct.unpack("<Q", f.read(8))
        for _ in range(n):
            cid, model, w, h = struct.unpack("<IiQQ", f.read(24))
            if model not in NUM_PARAMS:
                raise ValueError(f"unknown COLMAP camera model id {model}")
            out[cid] = Camera(cid, model, w, h, np.frombuffer(f.read(8 * NUM_PARAMS[model]), "<f8").copy())
    return out


def write_cameras(path: str, cameras: dict[int, Camera]) -> None:
    with open(path, "wb") as f:
        f.write(struct.pack("<Q", len(cameras)))
        for cid in sorted(cameras):
            c = cameras[cid]
            f.write(struct.pack("<IiQQ", c.camera_id, c.model_id, c.width, c.height))
            f.write(np.asarray(c.params[:NUM_PARAMS[c.model_id]], "<f8").tobytes())


def read_images(path: str) -> dict[int, Image]:
    out = {}
    with open(path, "rb") as f:
        buf = f.read()
    (n,) = struct.unpack_from("<Q", buf, 0)
    off = 8
    for _ in range(n):
        (iid,) = struct.unpack_from("<I", buf, off)
        q = np.frombuffer(buf, "<f8", 4, off + 4).copy()
        t = np.frombuffer(buf, "<f8", 3, off + 36).copy()
        (cid,) = struct.unpack_from("<I", buf, off + 60)
        end = buf.index(b"\0", off + 64)
        name = buf[off + 64:end].decode("utf-8")
        (m,) = struct.unpack_from("<Q", buf, end + 1)
        p = np.frombuffer(buf, _P2D, m, end + 9)
        out[iid] = Image(iid, q, t, cid, name, np.stack([p["x"], p["y"]], 1), p["id"].copy())
        off = end + 9 + m * _P2D.itemsize
    return out


def write_images(path: str, images: dict[int, Image]) -> None:
    with open(path, "wb") as f:
        f.write(struct.pack("<Q", len(images)))
        for iid in sorted(images):
            im = images[iid]
            f.write(struct.pack("<I", im.image_id))
            f.write(np.asarray(im.qvec_wxyz, "<f8").tobytes())
            f.write(np.asarray(im.tvec, "<f8").tobytes())
            f.write(struct.pack("<I", im.camera_id))
            f.write(im.name.encode("utf-8") + b"\0")
            m = len(im.xy)
            f.write(struct.pack("<Q", m))
            p = np.empty(m, _P2D)
            p["x"], p["y"], p["id"] = im.xy[:, 0], im.xy[:, 1], im.point3D_ids
            f.write(p.tobytes())


def read_points3D(path: str) -> dict[int, Point3D]:
    out = {}
    with open(path, "rb") as f:
        buf = f.read()
    (n,) = struct.unpack_from("<Q", buf, 0)
    off = 8
    for _ in range(n):
        (pid,) = struct.unpack_from("<Q", buf, off)
        xyz = np.frombuffer(buf, "<f8", 3, off + 8).copy()
        rgb = np.frombuffer(buf, "u1", 3, off + 32).copy()
        err, L = struct.unpack_from("<dQ", buf, off + 35)
        t = np.frombuffer(buf, _TRK, L, off + 51)
        out[pid] = Point3D(pid, xyz, rgb, err, t["image_id"].copy(), t["point2D_idx"].copy())
        off += 51 + L * _TRK.itemsize
    return out


def write_points3D(path: str, points: dict[int, Point3D]) -> None:
    with open(path, "wb") as f:
        f.write(struct.pack("<Q", len(points)))
        for pid in sorted(points):
            p = points[pid]
            f.write(struct.pack("<Q", p.point3D_id))
            f.write(np.asarray(p.xyz, "<f8").tobytes())
            f.write(np.asarray(p.rgb, "u1").tobytes())
            f.write(struct.pack("<dQ", float(p.error), len(p.image_ids)))
            t = np.empty(len(p.image_ids), _TRK)
            t["image_id"], t["point2D_idx"] = p.image_ids, p.point2D_idxs
            f.write(t.tobytes())


def read_model(path: str):
    return (read_cameras(os.path.join(path, "cameras.bin")), read_images(os.path.join(path, "images.bin")),
            read_points3D(os.path.join(path, "points3D.bin")))


def write_model(path: str, cameras, images, points) -> None:
    os.makedirs(path, exist_ok=True)
    write_cameras(os.path.join(path, "cameras.bin"), cameras)
    write_images(os.path.join(path, "images.bin"), images)
    write_points3D(os.path.join(path, "points3D.bin"), points)


# ---------------------------------------------------------------------------- model <-> flat scene
@dataclasses.dataclass
class ModelIndex:
    """What the flat scene forgets: ids, names, image sizes, the full feature tables and colours."""
    camera_ids: np.ndarray        # [K] sorted
    camera_size: np.ndarray       # [K,2]
    image_ids: np.ndarray         # [C] sorted
    image_names: list
    image_xy: list                # per image [m,2] all features (observed or not)
    point_ids: np.ndarray         # [P] sorted
    point_rgb: np.ndarray         # [P,3]
    obs_feature: np.ndarray       # [N] point2D_idx of every observation


def scene_from_model(cameras, images, points) -> tuple[S.Scene, ModelIndex]:
    """Sorted-id flattening (the order the C++ shim uses, glomap_b200/host/estimators_shim.h).  Track elements that
    refer to images absent from ``images`` are skipped (bundle_adjustment.cc:125)."""
    cam_ids = np.array(sorted(cameras), np.int64)
    img_ids = np.array(sorted(images), np.int64)
    pt_ids = np.array(sorted(points), np.uint64)
    for c in cameras.values():
        if c.model_id > 3:
            raise ValueError(f"camera model {c.model_id} is not supported by the BA kernels (models 0-3)")
    cidx = {int(c): i for i, c in enumerate(cam_ids)}
    iidx = {int(i): k for k, i in enumerate(img_ids)}
    K, C, P = len(cam_ids), len(img_ids), len(pt_ids)
    intr_model = np.array([cameras[int(c)].model_id for c in cam_ids], np.int32)
    intr = np.zeros((K, S.INTR_STRIDE))
    for k, c in enumerate(cam_ids):
        p = cameras[int(c)].params
        intr[k, :len(p)] = p
    quat, trans, cam_intr = np.empty((C, 4)), np.empty((C, 3)), np.empty(C, np.int32)
    for k, i in enumerate(img_ids):
        im = images[int(i)]
        quat[k] = [im.qvec_wxyz[1], im.qvec_wxyz[2], im.qvec_wxyz[3], im.qvec_wxyz[0]]   # COLMAP w x y z -> Eigen x y z w
        trans[k] = im.tvec
        cam_intr[k] = cidx[im.camera_id]
    pts = np.empty((P, 3))
    begin, obs_cam, obs_xy, obs_feat = [0], [], [], []
    for j, pid in enumerate(pt_ids):
        p = points[int(pid)]
        pts[j] = p.xyz
        for iid, fi in zip(p.image_ids, p.point2D_idxs):
            if int(iid) not in iidx:
                continue
            obs_cam.append(iidx[int(iid)]); obs_xy.append(images[int(iid)].xy[int(fi)]); obs_feat.append(int(fi))
        begin.append(len(obs_cam))
    scene = S.Scene(quat, trans, pts, np.asarray(begin, np.int64), np.asarray(obs_cam, np.int32),
                    np.asarray(obs_xy, np.float64).reshape(-1, 2), cam_intr, intr_model, intr)
    index = ModelIndex(cam_ids, np.array([[cameras[int(c)].width, cameras[int(c)].height] for c in cam_ids], np.int64),
                       img_ids, [images[int(i)].name for i in img_ids], [images[int(i)].xy for i in img_ids], pt_ids,
                       np.array([points[int(p)].rgb for p in pt_ids], np.uint8).reshape(-1, 3),
                       np.asarray(obs_feat, np.int64))
    return scene, index


def default_index(scene: S.Scene) -> ModelIndex:
    """Synthesised ids / feature tables: image i has exactly its observed features, in scene order."""
    C, P, K = scene.C, scene.P, len(scene.intr_model)
    order = np.argsort(scene.obs_cam, kind="stable")
    feat = np.empty(scene.N, np.int64)
    counts = np.bincount(scene.obs_cam, minlength=C)
    starts = np.concatenate([[0], np.cumsum(counts)])
    feat[order] = np.arange(scene.N) - np.repeat(starts[:-1], counts)
    xy_sorted = scene.obs_xy[order]
    return ModelIndex(np.arange(1, K + 1), np.zeros((K, 2), np.int64), np.arange(1, C + 1),
                      [f"image_{i + 1:06d}.jpg" for i in range(C)],
                      [xy_sorted[starts[i]:starts[i + 1]] for i in range(C)], np.arange(1, P + 1, dtype=np.uint64),
                      np.zeros((P, 3), np.uint8), feat)


def model_from_scene(scene: S.Scene, index: ModelIndex | None = None, min_supports: int = 2):
    """ConvertGlomapToColmap (colmap_converter.cc:22-133) for trivial frames."""
    C, P, K = scene.C, scene.P, len(scene.intr_model)
    if index is None:
        index = default_index(scene)
    cameras = {}
    for k in range(K):
        m = int(scene.intr_model[k])
        cameras[int(index.camera_ids[k])] = Camera(int(index.camera_ids[k]), m, int(index.camera_size[k, 0]),
                                                    int(index.camera_size[k, 1]), scene.intr_params[k, :NUM_PARAMS[m]].copy())
    p3d_ids = [np.full(len(index.image_xy[i]), INVALID_POINT3D, np.uint64) for i in range(C)]
    # mean reprojection error per point (Reconstruction::UpdatePoint3DErrors)
    from . import geometry as geo
    R = geo.quat_xyzw_to_rotmat(scene.quat)
    pt_of_obs = np.repeat(np.arange(P), np.diff(scene.pt_obs_begin))
    Xc = np.einsum("nij,nj->ni", R[scene.obs_cam], scene.points[pt_of_obs]) + scene.trans[scene.obs_cam]
    err = np.zeros(scene.N)
    ci = scene.cam_intr[scene.obs_cam]
    for k in range(K):
        mk = ci == k
        if mk.any():
            err[mk] = np.linalg.norm(S.project(int(scene.intr_model[k]), scene.intr_params[k], Xc[mk]) - scene.obs_xy[mk], axis=1)
    points = {}
    for j in range(P):
        a, b = int(scene.pt_obs_begin[j]), int(scene.pt_obs_begin[j + 1])
        if b - a < min_supports:
            continue
        pid = int(index.point_ids[j])
        img = index.image_ids[scene.obs_cam[a:b]].astype(np.uint32)
        points[pid] = Point3D(pid, scene.points[j].copy(), index.point_rgb[j].copy(), float(err[a:b].mean()), img,
                              index.obs_feature[a:b].astype(np.uint32))
        for o in range(a, b):
            p3d_ids[int(scene.obs_cam[o])][int(index.obs_feature[o])] = pid
    images = {}
    for i in range(C):
        q = scene.quat[i] / np.linalg.norm(scene.quat[i])
        images[int(index.image_ids[i])] = Image(int(index.image_ids[i]), np.array([q[3], q[0], q[1], q[2]]), scene.trans[i].copy(),
                                                int(index.camera_ids[scene.cam_intr[i]]), index.image_names[i],
                                                np.asarray(index.image_xy[i], np.float64).reshape(-1, 2), p3d_ids[i])
    return cameras, images, points


def write_clustered_model(out_dir: str, scene: S.Scene, index: ModelIndex | None, cluster_id, registered) -> list:
    """WriteGlomapReconstruction (io/colmap_io.cc:8-66) with the cluster filter of ConvertGlomapToColmap
    (colmap_converter.cc:22-131), trivial frames: ``cluster_id`` / ``registered`` [C] per image (the output of
    ``reconstruction_pruning.prune_weakly_connected_images``).  A model holds the images that stay registered in it:
    the reference deregisters every other frame before writing (colmap_converter.cc:122-128), and its tracks skip the
    images of those frames (:55-58, :86-90).  So if every id is -1, ``out_dir/0`` holds the registered images; otherwise
    ``out_dir/c`` holds the images of cluster c (all registered).  Track elements are restricted to the images written,
    points left with fewer than 2 elements are dropped, and every model keeps all cameras.  Camera models 0-3 only, as
    ``model_from_scene`` recomputes each point's mean reprojection error.  Returns the directories written."""
    from .mapper import compact_observations
    index = index if index is not None else default_index(scene)
    cid = np.asarray(cluster_id, np.int64)
    reg = np.asarray(registered, bool)
    img_ids = np.asarray(index.image_ids)
    if cid.max(initial=-1) == -1:
        jobs = [(os.path.join(out_dir, "0"), reg, reg)]
    else:
        jobs = [(os.path.join(out_dir, str(c)), cid == c, cid == c) for c in range(int(cid.max()) + 1)]
    written = []
    for path, keep_obs_img, keep_img in jobs:
        keep = keep_obs_img[scene.obs_cam]
        sub = compact_observations(scene, keep)
        sub_index = dataclasses.replace(index, obs_feature=np.asarray(index.obs_feature)[keep])
        cameras, images, points = model_from_scene(sub, sub_index)
        images = {int(i): images[int(i)] for i in img_ids[keep_img]}
        write_model(path, cameras, images, points)
        written.append(path)
    return written


# ---------------------------------------------------------------------------- command line
def _main(argv=None):
    """``python -m glomap_b200.colmap_io to-flat MODEL_DIR FLAT.bin`` converts a COLMAP sparse model into the flat
    binary problem of ``b200sfm_cli ba|gp`` (mapper_resume-style entry, exe/global_mapper.cc:110);
    ``from-flat MODEL_DIR FLAT.bin OUT_DIR`` writes the solved state back as a COLMAP model;
    ``prune MODEL_DIR OUT_DIR [--min_num_observations N]`` splits a model into its covisibility clusters on the GPU
    (PruneWeaklyConnectedImages, the ``mapper_resume --skip_pruning 0`` analogue for trivial frames) and writes one model
    per cluster to OUT_DIR/0, OUT_DIR/1, ...  Every subcommand reads camera models 0-3 (SIMPLE_PINHOLE, PINHOLE,
    SIMPLE_RADIAL, RADIAL) only: the flat problem holds those, and ``prune`` recomputes the points' reprojection errors of
    the models it writes.  The pruning itself does not read the intrinsics."""
    import argparse
    ap = argparse.ArgumentParser(prog="glomap_b200.colmap_io")
    sub = ap.add_subparsers(dest="cmd", required=True)
    a = sub.add_parser("to-flat"); a.add_argument("model"); a.add_argument("flat")
    b = sub.add_parser("from-flat"); b.add_argument("model"); b.add_argument("flat"); b.add_argument("out")
    c = sub.add_parser("prune", help="split into covisibility clusters (camera models 0-3)")
    c.add_argument("model"); c.add_argument("out")
    c.add_argument("--min_num_observations", type=int, default=0)
    args = ap.parse_args(argv)
    try:
        scene, index = scene_from_model(*read_model(args.model))
    except ValueError as e:
        raise SystemExit(f"{args.cmd}: {e} (colmap_io reads camera models 0-3 only)")
    if args.cmd == "prune":
        from .reconstruction_pruning import prune_weakly_connected_images
        out = prune_weakly_connected_images(scene.pt_obs_begin, scene.obs_cam, scene.C,
                                            min_num_observations=args.min_num_observations)
        for path in write_clustered_model(args.out, scene, index, out["cluster_id"], out["is_registered"]):
            print(f"wrote {path}")
        print(f"{out['num_clusters']} clusters, {int(out['is_registered'].sum())} of {scene.C} images registered")
    elif args.cmd == "to-flat":
        S.write_flat_problem(args.flat, scene)
        print(f"{scene.C} images, {scene.P} points, {scene.N} observations -> {args.flat}")
    else:
        solved = S.read_flat_problem(args.flat)
        if (solved.C, solved.P, solved.N) != (scene.C, scene.P, scene.N):
            raise SystemExit("flat problem does not match the model")
        write_model(args.out, *model_from_scene(solved, index))
        print(f"wrote {args.out}")


if __name__ == "__main__":
    _main()
