"""Flat problem  <->  COLMAP sparse model -- SURVEY.md 8(f) item 3.

The reference reads and writes its results through ``colmap::Reconstruction`` (glomap/io/colmap_io.cc:8-66,
glomap/io/colmap_converter.cc:22-209); COLMAP is not vendored, so the layouts are restated here from the public COLMAP
sources (src/colmap/scene/reconstruction_io*.cc, UPSTREAM-UNVERIFIED; binary files little-endian, packed):

  cameras.bin   u64 n | n x { u32 camera_id, i32 model_id, u64 width, u64 height, f64 params[num_params(model)] }
  images.bin    u64 n | n x { u32 image_id, f64 qvec[4] (w x y z), f64 tvec[3] (cam_from_world), u32 camera_id,
                              char name[] NUL-terminated, u64 m, m x { f64 x, f64 y, u64 point3D_id (2^64-1 = none) } }
  points3D.bin  u64 n | n x { u64 point3D_id, f64 xyz[3], u8 rgb[3], f64 error, u64 L, L x { u32 image_id, u32 point2D_idx } }
  rigs.bin      u64 n | n x { u32 rig_id, u32 num_sensors, [i32 ref_sensor_type, u32 ref_sensor_id  if num_sensors > 0],
                              (num_sensors - 1) x { i32 sensor_type, u32 sensor_id, u8 has_pose,
                                                    [f64 qvec[4] (w x y z), f64 tvec[3] (sensor_from_rig)  if has_pose] } }
  frames.bin    u64 n | n x { u32 frame_id, u32 rig_id, f64 qvec[4] (w x y z), f64 tvec[3] (rig_from_world),
                              u32 num_data_ids, num_data_ids x { i32 sensor_type, u32 sensor_id, u64 data_id } }

A rig is a reference sensor (identity sensor_from_rig) plus non-reference sensors, each with an optional
sensor_from_rig.  A frame is one capture of a rig: its rig_id, its rig_from_world and its data ids, one per image
(sensor_type 0 = CAMERA, sensor_id = the image's camera_id, data_id = its image_id).  frames.bin holds the frames that
have a pose (the registered ones); an image that no frame lists is not registered (Image::IsRegistered,
scene/image.h:65-66).  ``images.bin`` still stores every image's cam_from_world, composed as cam_from_rig *
rig_from_world for the registered ones, so that readers which ignore frames see the same poses.

The text layout (cameras.txt, images.txt, points3D.txt, rigs.txt, frames.txt) holds the same records, one per line,
after ``#`` comment lines, fields separated by spaces (images.txt: two lines per image, the second the m
``x y point3D_id`` triplets, -1 = none; rigs.txt / frames.txt: the sensor type as ``CAMERA``); floats are written
with 17 significant digits, so a model converted between the two formats keeps every bit.  Without rigs and frames,
a model is read as trivial rigs: one frame per image, every image registered.

``scene_from_model`` builds the SoA ``synthetic.Scene`` (trivial frames) or ``synthetic.RigScene`` (rigs and frames)
the C ABI consumes -- images, cameras, frames and points in sorted-id order (the order the C++ shim uses) -- plus a
``ModelIndex`` with everything needed to write the optimised state back, following ConvertColmapToGlomap
(colmap_converter.cc:133-209): a COLMAP sensor is a camera, so sensor k is camera k and has its own intrinsics block;
a frame is registered when it has a pose (:159); an image whose frame is not in the model gets a frame of its own,
not registered, with the rig of its camera; track colours are carried over (:196).  A non-reference sensor stored
without a pose is refused when an image of a registered frame uses it: global positioning throws on it in the reference
(Rig::SensorFromRig, global_positioning.cc:333), and rotation averaging, which would estimate it, does not run on a
resumed model.  Another such sensor is carried through unknown (``sensor_known`` False) and written back without a
pose.
``model_from_scene`` applies ConvertGlomapToColmap's rules: points with fewer than 2 supporting observations are
dropped (colmap_converter.cc:51,98), ``point3D_id`` is set on the observed features of the images kept, ``error`` is
the mean reprojection error (Reconstruction::UpdatePoint3DErrors).  Both conversions are vectorised over the
observations; only the parse of points3D, whose records have variable length, walks the points one by one."""
from __future__ import annotations

import dataclasses
import os
import struct

import numpy as np

from . import geometry as geo, synthetic as S

NUM_PARAMS = {0: 3, 1: 4, 2: 4, 3: 5, 4: 8, 5: 8, 6: 12, 7: 5, 8: 4, 9: 5, 10: 12, 11: 16}
MODEL_NAMES = {0: "SIMPLE_PINHOLE", 1: "PINHOLE", 2: "SIMPLE_RADIAL", 3: "RADIAL", 4: "OPENCV", 5: "OPENCV_FISHEYE",
               6: "FULL_OPENCV", 7: "FOV", 8: "SIMPLE_RADIAL_FISHEYE", 9: "RADIAL_FISHEYE", 10: "THIN_PRISM_FISHEYE",
               11: "RAD_TAN_THIN_PRISM_FISHEYE"}
SENSOR_CAMERA = 0                         # colmap::SensorType (INVALID = -1, CAMERA = 0, IMU = 1)
SENSOR_TYPES = {-1: "INVALID", 0: "CAMERA", 1: "IMU"}
INVALID_POINT3D = np.uint64(2**64 - 1)
_P2D = np.dtype([("x", "<f8"), ("y", "<f8"), ("id", "<u8")])
_TRK = np.dtype([("image_id", "<u4"), ("point2D_idx", "<u4")])
_DATA = np.dtype([("type", "<i4"), ("sensor_id", "<u4"), ("data_id", "<u8")])


class ModelError(ValueError):
    """A model that cannot be read or converted: a truncated or malformed file, or content the project does not
    support."""


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


@dataclasses.dataclass
class Rig:
    rig_id: int
    ref_sensor: tuple          # (sensor_type, sensor_id), or None for a rig without sensors
    sensors: list              # non-reference sensors: (sensor_type, sensor_id, qvec_wxyz | None, tvec | None)


@dataclasses.dataclass
class Frame:
    frame_id: int
    rig_id: int
    qvec_wxyz: np.ndarray      # rig_from_world
    tvec: np.ndarray
    data_ids: list             # (sensor_type, sensor_id, data_id)


# ---------------------------------------------------------------------------- raw model I/O
def _parse(path: str, parse):
    """``parse(buf)`` over the bytes of ``path``; a short or malformed file raises ModelError."""
    with open(path, "rb") as f:
        buf = f.read()
    try:
        return parse(buf)
    except ModelError:
        raise
    except (struct.error, ValueError, IndexError, UnicodeDecodeError) as e:
        raise ModelError(f"{path}: truncated or malformed ({e})") from None


def _check_model(model: int) -> int:
    if model not in NUM_PARAMS:
        raise ModelError(f"unknown COLMAP camera model id {model}")
    return model


def read_cameras(path: str) -> dict[int, Camera]:
    def parse(buf):
        out = {}
        (n,) = struct.unpack_from("<Q", buf, 0)
        off = 8
        for _ in range(n):
            cid, model, w, h = struct.unpack_from("<IiQQ", buf, off)
            k = NUM_PARAMS[_check_model(model)]
            out[cid] = Camera(cid, model, w, h, np.frombuffer(buf, "<f8", k, off + 24).copy())
            off += 24 + 8 * k
        return out
    return _parse(path, parse)


def write_cameras(path: str, cameras: dict[int, Camera]) -> None:
    with open(path, "wb") as f:
        f.write(struct.pack("<Q", len(cameras)))
        for cid in sorted(cameras):
            c = cameras[cid]
            f.write(struct.pack("<IiQQ", c.camera_id, c.model_id, c.width, c.height))
            f.write(np.asarray(c.params[:NUM_PARAMS[c.model_id]], "<f8").tobytes())


def read_images(path: str) -> dict[int, Image]:
    def parse(buf):
        out = {}
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
    return _parse(path, parse)


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
    def parse(buf):
        out = {}
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
    return _parse(path, parse)


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


def read_rigs(path: str) -> dict[int, Rig]:
    def parse(buf):
        out = {}
        (n,) = struct.unpack_from("<Q", buf, 0)
        off = 8
        for _ in range(n):
            rid, ns = struct.unpack_from("<II", buf, off)
            off += 8
            ref, sensors = None, []
            if ns > 0:
                ref = struct.unpack_from("<iI", buf, off)
                off += 8
            for _ in range(max(ns - 1, 0)):
                typ, sid, has = struct.unpack_from("<iIB", buf, off)
                off += 9
                q = t = None
                if has:
                    q = np.frombuffer(buf, "<f8", 4, off).copy()
                    t = np.frombuffer(buf, "<f8", 3, off + 32).copy()
                    off += 56
                sensors.append((typ, sid, q, t))
            out[rid] = Rig(rid, ref, sensors)
        return out
    return _parse(path, parse)


def write_rigs(path: str, rigs: dict[int, Rig]) -> None:
    with open(path, "wb") as f:
        f.write(struct.pack("<Q", len(rigs)))
        for rid in sorted(rigs):
            r = rigs[rid]
            f.write(struct.pack("<II", r.rig_id, 0 if r.ref_sensor is None else 1 + len(r.sensors)))
            if r.ref_sensor is not None:
                f.write(struct.pack("<iI", *r.ref_sensor))
            for typ, sid, q, t in r.sensors:
                f.write(struct.pack("<iIB", typ, sid, q is not None))
                if q is not None:
                    f.write(np.asarray(q, "<f8").tobytes() + np.asarray(t, "<f8").tobytes())


def read_frames(path: str) -> dict[int, Frame]:
    def parse(buf):
        out = {}
        (n,) = struct.unpack_from("<Q", buf, 0)
        off = 8
        for _ in range(n):
            fid, rid = struct.unpack_from("<II", buf, off)
            q = np.frombuffer(buf, "<f8", 4, off + 8).copy()
            t = np.frombuffer(buf, "<f8", 3, off + 40).copy()
            (m,) = struct.unpack_from("<I", buf, off + 64)
            d = np.frombuffer(buf, _DATA, m, off + 68)
            out[fid] = Frame(fid, rid, q, t, [(int(a), int(b), int(c)) for a, b, c in d.tolist()])
            off += 68 + m * _DATA.itemsize
        return out
    return _parse(path, parse)


def write_frames(path: str, frames: dict[int, Frame]) -> None:
    with open(path, "wb") as f:
        f.write(struct.pack("<Q", len(frames)))
        for fid in sorted(frames):
            fr = frames[fid]
            f.write(struct.pack("<II", fr.frame_id, fr.rig_id))
            f.write(np.asarray(fr.qvec_wxyz, "<f8").tobytes() + np.asarray(fr.tvec, "<f8").tobytes())
            d = np.array(fr.data_ids, np.int64).reshape(-1, 3)
            rec = np.empty(len(d), _DATA)
            rec["type"], rec["sensor_id"], rec["data_id"] = d[:, 0], d[:, 1], d[:, 2]
            f.write(struct.pack("<I", len(d)) + rec.tobytes())


# ---------------------------------------------------------------------------- text layout
def _g(values) -> str:
    return " ".join("%.17g" % v for v in values)


def _sensor_type(tok: str) -> int:
    names = {v: k for k, v in SENSOR_TYPES.items()}
    return names[tok] if tok in names else int(tok)


def _text_lines(path: str):
    with open(path, encoding="utf-8") as f:
        return [ln.rstrip("\n") for ln in f if ln.strip() and not ln.startswith("#")]


def _parse_text(path: str, parse):
    try:
        return parse(_text_lines(path))
    except ModelError:
        raise
    except (ValueError, IndexError, KeyError) as e:
        raise ModelError(f"{path}: truncated or malformed ({e!r})") from None


def _model_id(tok: str) -> int:
    names = {v: k for k, v in MODEL_NAMES.items()}
    return _check_model(names[tok] if tok in names else int(tok))


def read_cameras_text(path: str) -> dict[int, Camera]:
    def parse(lines):
        out = {}
        for ln in lines:
            e = ln.split()
            cid, model = int(e[0]), _model_id(e[1])
            p = np.array(e[4:], np.float64)
            if len(p) != NUM_PARAMS[model]:
                raise ModelError(f"{path}: truncated or malformed: camera {cid} has {len(p)} parameters, model {model} takes {NUM_PARAMS[model]}")
            out[cid] = Camera(cid, model, int(e[2]), int(e[3]), p)
        return out
    return _parse_text(path, parse)


def write_cameras_text(path: str, cameras: dict[int, Camera]) -> None:
    with open(path, "w", encoding="utf-8") as f:
        f.write("# Camera list with one line of data per camera:\n#   CAMERA_ID, MODEL, WIDTH, HEIGHT, PARAMS[]\n")
        for cid in sorted(cameras):
            c = cameras[cid]
            f.write(f"{c.camera_id} {MODEL_NAMES[c.model_id]} {c.width} {c.height} {_g(c.params[:NUM_PARAMS[c.model_id]])}\n")


def read_images_text(path: str) -> dict[int, Image]:
    def parse(lines):
        out = {}
        if len(lines) % 2:
            raise ModelError(f"{path}: truncated (an image line without its POINTS2D line)")
        for head, pts in zip(lines[0::2], lines[1::2]):
            e = head.split(maxsplit=9)
            iid = int(e[0])
            v = np.array(e[1:8], np.float64)
            tok = pts.split()
            if len(tok) % 3:
                raise ModelError(f"{path}: the points of image {iid} are truncated")
            xy = np.array(tok[0::3] + tok[1::3], np.float64).reshape(2, -1).T.copy()
            ids = np.array(tok[2::3], np.int64)
            out[iid] = Image(iid, v[:4], v[4:], int(e[8]), e[9], xy,
                             np.where(ids < 0, INVALID_POINT3D, ids.astype(np.uint64)).astype(np.uint64))
        return out
    with open(path, encoding="utf-8") as f:                 # the POINTS2D line of an image without features is empty
        lines = [ln.rstrip("\n") for ln in f if not ln.startswith("#")]
    try:
        return parse(lines)
    except ModelError:
        raise
    except (ValueError, IndexError) as e:
        raise ModelError(f"{path}: truncated or malformed ({e!r})") from None


def write_images_text(path: str, images: dict[int, Image]) -> None:
    with open(path, "w", encoding="utf-8") as f:
        f.write("# Image list with two lines of data per image:\n#   IMAGE_ID, QW, QX, QY, QZ, TX, TY, TZ, CAMERA_ID, NAME\n"
                "#   POINTS2D[] as (X, Y, POINT3D_ID)\n")
        for iid in sorted(images):
            im = images[iid]
            f.write(f"{im.image_id} {_g(im.qvec_wxyz)} {_g(im.tvec)} {im.camera_id} {im.name}\n")
            ids = np.asarray(im.point3D_ids, np.uint64)
            sid = np.where(ids == INVALID_POINT3D, -1, ids.astype(np.int64))
            f.write(" ".join(f"{x:.17g} {y:.17g} {i}" for (x, y), i in zip(np.asarray(im.xy).tolist(), sid.tolist())) + "\n")


def read_points3D_text(path: str) -> dict[int, Point3D]:
    def parse(lines):
        out = {}
        for ln in lines:
            e = ln.split()
            pid = int(e[0])
            trk = np.array(e[8:], np.int64)
            if len(trk) % 2:
                raise ModelError(f"{path}: the track of point {pid} is truncated")
            out[pid] = Point3D(pid, np.array(e[1:4], np.float64), np.array(e[4:7], np.uint8), float(e[7]),
                               trk[0::2].astype(np.uint32), trk[1::2].astype(np.uint32))
        return out
    return _parse_text(path, parse)


def write_points3D_text(path: str, points: dict[int, Point3D]) -> None:
    with open(path, "w", encoding="utf-8") as f:
        f.write("# 3D point list with one line of data per point:\n"
                "#   POINT3D_ID, X, Y, Z, R, G, B, ERROR, TRACK[] as (IMAGE_ID, POINT2D_IDX)\n")
        for pid in sorted(points):
            p = points[pid]
            trk = np.stack([np.asarray(p.image_ids, np.int64), np.asarray(p.point2D_idxs, np.int64)], 1).ravel()
            f.write(f"{p.point3D_id} {_g(p.xyz)} {' '.join(str(int(c)) for c in p.rgb)} {float(p.error):.17g} "
                    f"{' '.join(map(str, trk.tolist()))}\n")


def read_rigs_text(path: str) -> dict[int, Rig]:
    def parse(lines):
        out = {}
        for ln in lines:
            e = ln.split()
            rid, ns = int(e[0]), int(e[1])
            ref, sensors, k = None, [], 2
            if ns > 0:
                ref, k = (_sensor_type(e[2]), int(e[3])), 4
            for _ in range(max(ns - 1, 0)):
                typ, sid, has = _sensor_type(e[k]), int(e[k + 1]), int(e[k + 2])
                k += 3
                q = t = None
                if has:
                    v = np.array(e[k:k + 7], np.float64)
                    if len(v) != 7:
                        raise ModelError(f"{path}: the pose of sensor {sid} of rig {rid} is truncated")
                    q, t = v[:4], v[4:]
                    k += 7
                sensors.append((typ, sid, q, t))
            out[rid] = Rig(rid, ref, sensors)
        return out
    return _parse_text(path, parse)


def write_rigs_text(path: str, rigs: dict[int, Rig]) -> None:
    with open(path, "w", encoding="utf-8") as f:
        f.write("# Rig calib list with one line of data per calib:\n#   RIG_ID, NUM_SENSORS, REF_SENSOR_TYPE, REF_SENSOR_ID, "
                "SENSORS[] as (SENSOR_TYPE, SENSOR_ID, HAS_POSE, [QW, QX, QY, QZ, TX, TY, TZ])\n")
        for rid in sorted(rigs):
            r = rigs[rid]
            e = [str(r.rig_id), str(0 if r.ref_sensor is None else 1 + len(r.sensors))]
            if r.ref_sensor is not None:
                e += [SENSOR_TYPES[r.ref_sensor[0]], str(r.ref_sensor[1])]
            for typ, sid, q, t in r.sensors:
                e += [SENSOR_TYPES[typ], str(sid), "1" if q is not None else "0"]
                if q is not None:
                    e += [_g(q), _g(t)]
            f.write(" ".join(e) + "\n")


def read_frames_text(path: str) -> dict[int, Frame]:
    def parse(lines):
        out = {}
        for ln in lines:
            e = ln.split()
            fid, rid = int(e[0]), int(e[1])
            v = np.array(e[2:9], np.float64)
            m = int(e[9])
            d = e[10:]
            if len(d) != 3 * m:
                raise ModelError(f"{path}: the data ids of frame {fid} are truncated")
            out[fid] = Frame(fid, rid, v[:4], v[4:], [(_sensor_type(d[3 * i]), int(d[3 * i + 1]), int(d[3 * i + 2]))
                                                      for i in range(m)])
        return out
    return _parse_text(path, parse)


def write_frames_text(path: str, frames: dict[int, Frame]) -> None:
    with open(path, "w", encoding="utf-8") as f:
        f.write("# Frame list with one line of data per frame:\n#   FRAME_ID, RIG_ID, RIG_FROM_WORLD[QW, QX, QY, QZ, TX, TY, "
                "TZ], NUM_DATA_IDS, DATA_IDS[] as (SENSOR_TYPE, SENSOR_ID, DATA_ID)\n")
        for fid in sorted(frames):
            fr = frames[fid]
            d = " ".join(f"{SENSOR_TYPES[a]} {b} {c}" for a, b, c in fr.data_ids)
            f.write(f"{fr.frame_id} {fr.rig_id} {_g(fr.qvec_wxyz)} {_g(fr.tvec)} {len(fr.data_ids)} {d}".rstrip() + "\n")


_READERS = {"bin": (read_cameras, read_images, read_points3D, read_rigs, read_frames),
            "txt": (read_cameras_text, read_images_text, read_points3D_text, read_rigs_text, read_frames_text)}
_WRITERS = {"bin": (write_cameras, write_images, write_points3D, write_rigs, write_frames),
            "txt": (write_cameras_text, write_images_text, write_points3D_text, write_rigs_text, write_frames_text)}
_FILES = ("cameras", "images", "points3D", "rigs", "frames")


def model_format(path: str) -> str:
    """``bin`` or ``txt``: the layout of the model in ``path`` (binary first, as Reconstruction::Read)."""
    for fmt in ("bin", "txt"):
        if all(os.path.isfile(os.path.join(path, f"{n}.{fmt}")) for n in _FILES[:3]):
            return fmt
    raise ModelError(f"{path}: no COLMAP model (cameras, images and points3D .bin or .txt)")


def read_model(path: str):
    """(cameras, images, points) of the binary or text model in ``path``."""
    fmt = model_format(path)
    return tuple(r(os.path.join(path, f"{n}.{fmt}")) for r, n in zip(_READERS[fmt][:3], _FILES[:3]))


def read_rigs_frames(path: str):
    """(rigs, frames) of the model in ``path``, or (None, None) when it has neither (trivial rigs)."""
    fmt = model_format(path)
    have = [os.path.isfile(os.path.join(path, f"{n}.{fmt}")) for n in _FILES[3:]]
    if not any(have):
        return None, None
    if not all(have):
        raise ModelError(f"{path}: rigs.{fmt} and frames.{fmt} come together; one is missing")
    return tuple(r(os.path.join(path, f"{n}.{fmt}")) for r, n in zip(_READERS[fmt][3:], _FILES[3:]))


def write_model(path: str, cameras, images, points, rigs=None, frames=None, fmt: str = "bin") -> None:
    """Writes the model in the ``bin`` or ``txt`` layout; rigs and frames only when given."""
    os.makedirs(path, exist_ok=True)
    parts = (cameras, images, points) + (() if rigs is None else (rigs, frames))
    for w, n, part in zip(_WRITERS[fmt], _FILES, parts):
        w(os.path.join(path, f"{n}.{fmt}"), part)


# ---------------------------------------------------------------------------- model <-> flat scene
@dataclasses.dataclass
class ModelIndex:
    """What the flat scene forgets: ids, names, image sizes, the full feature tables and colours; for rigs the rig
    and frame ids, the record order of the rigs' sensors, the input registration and the input image poses."""
    camera_ids: np.ndarray        # [K] sorted (rigs: [S], sensor k = camera k)
    camera_size: np.ndarray       # [K,2]
    image_ids: np.ndarray         # [C] sorted (rigs: [I], the image table)
    image_names: list
    image_xy: list                # per image [m,2] all features (observed or not)
    point_ids: np.ndarray         # [P] sorted
    point_rgb: np.ndarray         # [P,3]
    obs_feature: np.ndarray       # [N] point2D_idx of every observation
    rig_ids: np.ndarray | None = None          # [R] sorted
    rig_sensors: list | None = None            # per rig: its non-reference sensors, in record order
    frame_ids: np.ndarray | None = None        # [F] (-1: the frame of an image no frame lists)
    frame_registered: np.ndarray | None = None  # [F] the frame had a pose in the model
    image_pose: np.ndarray | None = None       # [I,7] cam_from_world as read (qw qx qy qz tx ty tz)


def _sorted_ids(d: dict, dtype=np.int64) -> np.ndarray:
    return np.array(sorted(d), dtype) if d else np.zeros(0, dtype)


def _lookup(sorted_ids: np.ndarray, ids: np.ndarray):
    """(index, found) of ``ids`` in ``sorted_ids``."""
    ids = np.asarray(ids, np.int64)
    k = np.searchsorted(sorted_ids, ids)
    kc = np.minimum(k, max(len(sorted_ids) - 1, 0))
    found = (k < len(sorted_ids)) & (sorted_ids[kc] == ids) if len(sorted_ids) else np.zeros(len(ids), bool)
    return kc, found


def _wxyz_to_xyzw(q) -> np.ndarray:
    q = np.asarray(q, np.float64).reshape(-1, 4)
    return q[:, [1, 2, 3, 0]]


def scene_from_model(cameras, images, points, rigs=None, frames=None):
    """Sorted-id flattening (the order the C++ shim uses, glomap_b200/host/estimators_shim.h): (scene, index).
    Without ``rigs`` / ``frames`` the scene is a ``synthetic.Scene``, one camera per image; with them a
    ``synthetic.RigScene`` whose sensors are the cameras and whose frames are those of ``frames`` (sorted ids) followed
    by one unregistered frame per image that no frame lists (see the module docstring; ``index.frame_registered``).
    Track elements that refer to images absent from ``images`` are skipped (bundle_adjustment.cc:125)."""
    if (rigs is None) != (frames is None):
        raise ModelError("rigs and frames come together")
    cam_ids = _sorted_ids(cameras)
    img_ids = _sorted_ids(images)
    pt_ids = _sorted_ids(points, np.uint64)
    for c in cameras.values():
        if c.model_id > 3:
            raise ModelError(f"camera model {c.model_id} is not supported by the BA kernels (models 0-3)")
    K, C, P = len(cam_ids), len(img_ids), len(pt_ids)
    intr_model = np.array([cameras[int(c)].model_id for c in cam_ids], np.int32)
    intr = np.zeros((K, S.INTR_STRIDE))
    for k, c in enumerate(cam_ids):
        p = cameras[int(c)].params
        intr[k, :len(p)] = p
    ims = [images[int(i)] for i in img_ids]
    qv = np.array([im.qvec_wxyz for im in ims], np.float64).reshape(-1, 4)
    trans = np.array([im.tvec for im in ims], np.float64).reshape(-1, 3)
    cam_intr, cam_found = _lookup(cam_ids, [im.camera_id for im in ims])
    if not cam_found.all():
        raise ModelError(f"image {int(img_ids[~cam_found][0])} names a camera the model does not have")
    # the feature tables, concatenated: feature f of image i is row feat_begin[i] + f
    nfeat = np.array([len(im.xy) for im in ims], np.int64)
    feat_begin = np.concatenate([[0], np.cumsum(nfeat)])
    all_xy = np.concatenate([np.asarray(im.xy, np.float64).reshape(-1, 2) for im in ims]) if C else np.zeros((0, 2))
    # the tracks, concatenated (one pass over the point records)
    pts_rec = [points[int(p)] for p in pt_ids]
    lens = np.fromiter((len(p.image_ids) for p in pts_rec), np.int64, P)
    el_img = np.concatenate([p.image_ids for p in pts_rec]).astype(np.int64) if P else np.zeros(0, np.int64)
    el_feat = np.concatenate([p.point2D_idxs for p in pts_rec]).astype(np.int64) if P else np.zeros(0, np.int64)
    xyz = np.array([p.xyz for p in pts_rec], np.float64).reshape(-1, 3)
    rgb = np.array([p.rgb for p in pts_rec], np.uint8).reshape(-1, 3)
    obs_img, keep = _lookup(img_ids, el_img)
    obs_img, feat = obs_img[keep], el_feat[keep]
    bad = feat >= nfeat[obs_img]
    if bad.any():
        raise ModelError(f"a track element names feature {int(feat[bad][0])} of image {int(img_ids[obs_img[bad][0]])}, "
                         f"which has {int(nfeat[obs_img[bad][0]])}")
    pt_of_el = np.repeat(np.arange(P), lens)
    begin = np.concatenate([[0], np.cumsum(np.bincount(pt_of_el[keep], minlength=P))]).astype(np.int64)
    obs_xy = all_xy[feat_begin[obs_img] + feat].reshape(-1, 2)
    size = np.array([[cameras[int(c)].width, cameras[int(c)].height] for c in cam_ids], np.int64).reshape(-1, 2)
    index = ModelIndex(cam_ids, size, img_ids, [im.name for im in ims], [im.xy for im in ims], pt_ids, rgb, feat)
    if rigs is None:
        quat = _wxyz_to_xyzw(qv)                                  # COLMAP w x y z -> Eigen x y z w
        scene = S.Scene(quat, trans, xyz, begin, obs_img.astype(np.int32), obs_xy, cam_intr.astype(np.int32),
                        intr_model, intr)
        return scene, index
    return _rig_scene(cameras, rigs, frames, index, qv, trans, cam_intr, intr_model, intr, xyz, begin, obs_img, obs_xy)


def _rig_scene(cameras, rigs, frames, index, qv, trans, img_sensor, intr_model, intr, xyz, begin, obs_img, obs_xy):
    """The RigScene half of ``scene_from_model`` (ConvertColmapToGlomap, colmap_converter.cc:148-179)."""
    cam_ids, img_ids = index.camera_ids, index.image_ids
    K, I = len(cam_ids), len(img_ids)
    rig_ids = _sorted_ids(rigs)
    sensor_rig = np.full(K, -1, np.int32)
    ref_sensor = np.full(len(rig_ids), -1, np.int32)
    s_quat, s_trans = np.tile([0.0, 0, 0, 1], (K, 1)), np.zeros((K, 3))
    known = np.ones(K, bool)
    rig_sensors = []
    for r, rid in enumerate(rig_ids):
        rig = rigs[int(rid)]
        members = ([] if rig.ref_sensor is None else [rig.ref_sensor]) + [(t, s) for t, s, _, _ in rig.sensors]
        for typ, sid in members:
            if typ != SENSOR_CAMERA:
                raise ModelError(f"rig {int(rid)} has a sensor of type {SENSOR_TYPES.get(typ, typ)}; only cameras are supported")
            k, ok = _lookup(cam_ids, [sid])
            if not ok[0]:
                raise ModelError(f"rig {int(rid)} names camera {sid}, which the model does not have")
            if sensor_rig[k[0]] >= 0:
                raise ModelError(f"camera {sid} is a sensor of two rigs")
            sensor_rig[k[0]] = r
        if rig.ref_sensor is not None:
            ref_sensor[r] = _lookup(cam_ids, [rig.ref_sensor[1]])[0][0]
        order = []
        for typ, sid, q, t in rig.sensors:
            k = int(_lookup(cam_ids, [sid])[0][0])
            if q is None:
                known[k] = False
            else:
                s_quat[k], s_trans[k] = _wxyz_to_xyzw(q)[0], t
            order.append(k)
        rig_sensors.append(order)
    used = np.unique(img_sensor)
    if (sensor_rig[used] < 0).any():
        raise ModelError(f"camera {int(cam_ids[used[sensor_rig[used] < 0][0]])} is not a sensor of any rig")
    frame_ids = _sorted_ids(frames)
    image_frame = np.full(I, -1, np.int64)
    frame_rig = np.empty(len(frame_ids), np.int32)
    for f, fid in enumerate(frame_ids):
        fr = frames[int(fid)]
        r, ok = _lookup(rig_ids, [fr.rig_id])
        if not ok[0]:
            raise ModelError(f"frame {int(fid)} names rig {fr.rig_id}, which the model does not have")
        frame_rig[f] = r[0]
        d = np.array(fr.data_ids, np.int64).reshape(-1, 3)
        k, ok = _lookup(img_ids, d[:, 2])
        if not ok.all() or (d[:, 0] != SENSOR_CAMERA).any():
            raise ModelError(f"frame {int(fid)} lists data that is not an image of the model")
        if (cam_ids[img_sensor[k]] != d[:, 1]).any() or (sensor_rig[img_sensor[k]] != r[0]).any():
            raise ModelError(f"frame {int(fid)} lists an image whose camera is not the named sensor of its rig")
        if (image_frame[k] >= 0).any() or len(np.unique(img_sensor[k])) != len(k):
            raise ModelError(f"frame {int(fid)} lists an image twice, or two images of one sensor")
        image_frame[k] = f
    orphan = np.flatnonzero(image_frame < 0)
    F0 = len(frame_ids)
    # global positioning reads the sensor_from_rig of every registered image (Rig::SensorFromRig throws without one,
    # global_positioning.cc:333), and rotation averaging, which would estimate it, does not run on a resumed model
    bad = ~known[img_sensor[image_frame >= 0]]
    if bad.any():
        k = int(img_sensor[image_frame >= 0][bad][0])
        raise ModelError(f"sensor {int(cam_ids[k])} of rig {int(rig_ids[sensor_rig[k]])} has no sensor_from_rig but "
                         "images of registered frames use it; resuming needs their pose")
    image_frame[orphan] = F0 + np.arange(len(orphan))
    # rig_from_world of the registered frames; an image no frame lists gets sensor_from_rig^-1 * cam_from_world
    fq = _wxyz_to_xyzw([frames[int(i)].qvec_wxyz for i in frame_ids]) if F0 else np.zeros((0, 4))
    ft = np.array([frames[int(i)].tvec for i in frame_ids], np.float64).reshape(-1, 3)
    so = img_sensor[orphan]
    Rs = geo.quat_xyzw_to_rotmat(s_quat[so]).reshape(-1, 3, 3)
    Rc = geo.quat_xyzw_to_rotmat(_wxyz_to_xyzw(qv[orphan])).reshape(-1, 3, 3)
    Ro = np.einsum("nji,njk->nik", Rs, Rc)
    to = np.einsum("nji,nj->ni", Rs, trans[orphan] - s_trans[so])
    quat = np.concatenate([fq, geo.rotmat_to_quat_xyzw_fast(Ro) if len(orphan) else np.zeros((0, 4))])
    ftrans = np.concatenate([ft, to])
    frame_rig = np.concatenate([frame_rig, sensor_rig[so]]).astype(np.int32)
    scene = S.RigScene(quat, ftrans, xyz, begin, image_frame[obs_img].astype(np.int32),
                       img_sensor[obs_img].astype(np.uint16), obs_xy, s_quat, s_trans, np.arange(K, dtype=np.int32),
                       intr_model, intr, image_frame.astype(np.int32), img_sensor.astype(np.int32), frame_rig,
                       sensor_rig, ref_sensor, known)
    index.rig_ids, index.rig_sensors = rig_ids, rig_sensors
    index.frame_ids = np.concatenate([frame_ids, np.full(len(orphan), -1, np.int64)])
    index.frame_registered = np.arange(scene.F) < F0
    index.image_pose = np.concatenate([qv, trans], 1)
    return scene, index


def _image_scene(scene: S.RigScene) -> S.Scene:
    """The rig problem as a trivial-frame Scene over its images (poses composed), with one intrinsics block per
    sensor: the camera of image k is its sensor."""
    out = scene.images_scene()
    out.cam_intr = scene.image_sensor.astype(np.int32)
    out.intr_model = scene.intr_model[scene.sensor_intr].copy()
    out.intr_params = scene.intr_params[scene.sensor_intr].copy()
    return out


def default_index(scene) -> ModelIndex:
    """Synthesised ids / feature tables: image i has exactly its observed features, in scene order.  For a RigScene:
    camera = sensor, ids 1, 2, ... for rigs, frames and images, every frame registered."""
    if isinstance(scene, S.RigScene):
        index = default_index(_image_scene(scene))
        ref = scene.sensor_is_ref
        index.rig_ids = np.arange(1, len(scene.rig_ref_sensor) + 1)
        index.rig_sensors = [list(np.flatnonzero((scene.sensor_rig == r) & ~ref)) for r in range(len(scene.rig_ref_sensor))]
        index.frame_ids = np.arange(1, scene.F + 1)
        index.frame_registered = np.ones(scene.F, bool)
        return index
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


def _wxyz(q_xyzw) -> np.ndarray:
    q = np.asarray(q_xyzw, np.float64).reshape(-1, 4)
    q = q / np.linalg.norm(q, axis=1, keepdims=True)
    return q[:, [3, 0, 1, 2]]


def model_from_scene(scene, index: ModelIndex | None = None, min_supports: int = 2, frame_registered=None):
    """ConvertGlomapToColmap (colmap_converter.cc:22-131).  A Scene gives (cameras, images, points); a RigScene gives
    (cameras, images, points, rigs, frames): one camera per sensor, every rig, the frames of ``frame_registered``
    ([F], default ``index.frame_registered``) with their rig_from_world, and every image -- those of a registered frame
    with cam_from_rig * rig_from_world and their observations, the others with their input pose (``index.image_pose``)
    and no observation."""
    if index is None:
        index = default_index(scene)
    if isinstance(scene, S.RigScene):
        return _rig_model(scene, index, min_supports, frame_registered)
    C, P, K = scene.C, scene.P, len(scene.intr_model)
    cameras = {}
    for k in range(K):
        m = int(scene.intr_model[k])
        cameras[int(index.camera_ids[k])] = Camera(int(index.camera_ids[k]), m, int(index.camera_size[k, 0]),
                                                    int(index.camera_size[k, 1]), scene.intr_params[k, :NUM_PARAMS[m]].copy())
    # mean reprojection error per point (Reconstruction::UpdatePoint3DErrors)
    R = geo.quat_xyzw_to_rotmat(scene.quat)
    lens = np.diff(scene.pt_obs_begin)
    pt_of_obs = np.repeat(np.arange(P), lens)
    Xc = np.einsum("nij,nj->ni", R[scene.obs_cam], scene.points[pt_of_obs]) + scene.trans[scene.obs_cam]
    err = np.zeros(scene.N)
    ci = scene.cam_intr[scene.obs_cam]
    for k in range(K):
        mk = ci == k
        if mk.any():
            err[mk] = np.linalg.norm(S.project(int(scene.intr_model[k]), scene.intr_params[k], Xc[mk]) - scene.obs_xy[mk], axis=1)
    # point3D_id of every feature: the features of all images concatenated, then split per image
    nfeat = np.array([len(xy) for xy in index.image_xy], np.int64)
    feat_begin = np.concatenate([[0], np.cumsum(nfeat)])
    ids = np.full(int(feat_begin[-1]), INVALID_POINT3D, np.uint64)
    obs_feature = np.asarray(index.obs_feature, np.int64)
    kept = (lens >= min_supports)[pt_of_obs]
    ids[feat_begin[scene.obs_cam[kept]] + obs_feature[kept]] = np.asarray(index.point_ids, np.uint64)[pt_of_obs[kept]]
    img_of_obs = np.asarray(index.image_ids)[scene.obs_cam].astype(np.uint32)
    feat_of_obs = obs_feature.astype(np.uint32)
    points = {}
    for j in np.flatnonzero(lens >= min_supports):
        a, b = int(scene.pt_obs_begin[j]), int(scene.pt_obs_begin[j + 1])
        pid = int(index.point_ids[j])
        points[pid] = Point3D(pid, scene.points[j].copy(), index.point_rgb[j].copy(), float(err[a:b].mean()),
                              img_of_obs[a:b], feat_of_obs[a:b])
    images = {}
    for i in range(C):
        q = scene.quat[i] / np.linalg.norm(scene.quat[i])
        images[int(index.image_ids[i])] = Image(int(index.image_ids[i]), np.array([q[3], q[0], q[1], q[2]]), scene.trans[i].copy(),
                                                int(index.camera_ids[scene.cam_intr[i]]), index.image_names[i],
                                                np.asarray(index.image_xy[i], np.float64).reshape(-1, 2),
                                                ids[feat_begin[i]:feat_begin[i + 1]])
    return cameras, images, points


def _rig_model(scene: S.RigScene, index: ModelIndex, min_supports: int, frame_registered):
    reg = np.asarray(index.frame_registered if frame_registered is None else frame_registered, bool)
    from .mapper import compact_observations
    sub = compact_observations(_image_scene(scene), reg[scene.obs_frame])
    sub_index = dataclasses.replace(index, obs_feature=np.asarray(index.obs_feature)[reg[scene.obs_frame]])
    cameras, images, points = model_from_scene(sub, sub_index, min_supports)
    cam_ids = np.asarray(index.camera_ids)
    if index.image_pose is not None:                        # an image of an unregistered frame keeps its input pose
        for k in np.flatnonzero(~reg[scene.image_frame]):
            im = images[int(index.image_ids[k])]
            im.qvec_wxyz, im.tvec = index.image_pose[k, :4].copy(), index.image_pose[k, 4:].copy()
    sq = _wxyz(scene.sensor_quat)
    rigs = {}
    for r, rid in enumerate(np.asarray(index.rig_ids)):
        s0 = int(scene.rig_ref_sensor[r])
        ref = None if s0 < 0 else (SENSOR_CAMERA, int(cam_ids[s0]))
        rigs[int(rid)] = Rig(int(rid), ref, [(SENSOR_CAMERA, int(cam_ids[s]), sq[s].copy() if scene.sensor_known[s] else None,
                                              scene.sensor_trans[s].copy() if scene.sensor_known[s] else None)
                                             for s in index.rig_sensors[r]])
    fq = _wxyz(scene.quat)
    frames = {}
    img_ids = np.asarray(index.image_ids)
    order = np.argsort(scene.image_frame, kind="stable")
    fb = np.concatenate([[0], np.cumsum(np.bincount(scene.image_frame, minlength=scene.F))])
    for f in np.flatnonzero(reg):
        fid = int(index.frame_ids[f])
        if fid < 0:
            raise ValueError("a frame made for an image that no frame lists has no id and cannot be registered")
        imgs = order[fb[f]:fb[f + 1]]
        frames[fid] = Frame(fid, int(index.rig_ids[scene.frame_rig[f]]), fq[f].copy(), scene.trans[f].copy(),
                            [(SENSOR_CAMERA, int(cam_ids[scene.image_sensor[k]]), int(img_ids[k])) for k in imgs])
    return cameras, images, points, rigs, frames


def _obs_keys(scene) -> np.ndarray:
    """[N,3] int64 (point * images + image, x bits, y bits) of every observation."""
    rig = isinstance(scene, S.RigScene)
    img = scene.obs_image() if rig else scene.obs_cam
    n = scene.I if rig else scene.C
    pt = np.repeat(np.arange(scene.P, dtype=np.int64), np.diff(scene.pt_obs_begin))
    xy = np.ascontiguousarray(scene.obs_xy, np.float64).view(np.int64).reshape(-1, 2)
    return np.column_stack([pt * n + np.asarray(img, np.int64), xy])


def _ranked(keys: np.ndarray) -> np.ndarray:
    """``keys`` with a column appended: the occurrence number of each row among the equal rows before it."""
    order = np.lexsort(keys.T[::-1])
    k = keys[order]
    first = np.r_[True, (k[1:] != k[:-1]).any(axis=1)] if len(k) else np.zeros(0, bool)
    pos = np.arange(len(k))
    rank = np.empty(len(k), np.int64)
    rank[order] = pos - np.maximum.accumulate(np.where(first, pos, 0))
    return np.column_stack([keys, rank])


def reindex_observations(index: ModelIndex, before, after) -> ModelIndex:
    """``index`` for ``after``, a scene whose observations are a subset of those of ``before`` (the scene ``index``
    was made for): what the mapper's filters and its compaction to the registered images leave.  Each observation of
    ``after`` is found in ``before`` by its point, image and pixel, and takes that observation's feature index.  Two
    elements of one track in one image at the same pixel are told apart by their order: every filter decides them
    alike (they have the same residual, angle and track), so both survive or neither does, in the same order."""
    kin, kout = _ranked(_obs_keys(before)), _ranked(_obs_keys(after))
    n_in = len(kin)
    keys = np.concatenate([kin, kout])
    flag = np.r_[np.zeros(n_in, np.int8), np.ones(len(kout), np.int8)]
    order = np.lexsort((flag, keys[:, 3], keys[:, 2], keys[:, 1], keys[:, 0]))
    is_in = flag[order] == 0
    last_in = np.maximum.accumulate(np.where(is_in, np.arange(len(order)), -1))   # sorted position of the last input
    pos = np.flatnonzero(~is_in)
    found = last_in[pos] >= 0
    match = order[np.maximum(last_in[pos], 0)]
    if not found.all() or (keys[match] != keys[order[pos]]).any():
        raise ValueError("the scene has observations that the indexed scene does not have")
    feat = np.empty(len(kout), np.int64)
    feat[order[pos] - n_in] = np.asarray(index.obs_feature, np.int64)[match]
    return dataclasses.replace(index, obs_feature=feat)


def write_clustered_model(out_dir: str, scene, index: ModelIndex | None, cluster_id, registered, fmt: str = "bin") -> list:
    """WriteGlomapReconstruction (io/colmap_io.cc:8-66) with the cluster filter of ConvertGlomapToColmap
    (colmap_converter.cc:22-131), in frame space: ``cluster_id`` / ``registered`` hold one entry per frame -- per image
    of a ``Scene`` (trivial frames), per frame of a ``RigScene`` (``frame_cluster_id`` / ``frame_registered`` of the
    mapper, or the output of ``reconstruction_pruning.prune_weakly_connected_images``).  If every id is -1,
    ``out_dir/0`` is written; otherwise ``out_dir/c`` for every cluster c.  Model c keeps the frames the reference does
    not deregister (:122-128): those of cluster c that are registered, and, by the reference's ``cluster_id != 0`` rule,
    the unregistered frames of cluster 0 too; with every id -1, the registered frames.  Track elements are those of the
    registered frames of the model (:55-58, :86-90); points left with fewer than 2 are dropped.  The model holds the
    images of its frames -- and, with every id -1 on a RigScene, also the images of the unregistered frames, with their
    input pose and no observation (only the rig layout can hold an image without a registered frame) -- and every
    camera and rig.  Camera models 0-3 only, as ``model_from_scene`` recomputes each point's mean reprojection error.
    Returns the directories written."""
    from .mapper import compact_observations
    rig = isinstance(scene, S.RigScene)
    index = index if index is not None else default_index(scene)
    cid = np.asarray(cluster_id, np.int64)
    reg = np.asarray(registered, bool)
    if cid.max(initial=-1) == -1:
        jobs = [(os.path.join(out_dir, "0"), reg, reg)]
    else:
        jobs = [(os.path.join(out_dir, str(c)), (cid == c) & reg, (cid == c) & (reg | (c == 0)))
                for c in range(int(cid.max()) + 1)]
    obs_frame = scene.obs_frame if rig else scene.obs_cam
    img_frame = scene.image_frame if rig else np.arange(scene.C)
    img_ids = np.asarray(index.image_ids)
    written = []
    for path, keep_obs_frame, keep_frame in jobs:
        keep = keep_obs_frame[obs_frame]
        sub = compact_observations(scene, keep)
        sub_index = dataclasses.replace(index, obs_feature=np.asarray(index.obs_feature)[keep])
        model = model_from_scene(sub, sub_index, frame_registered=keep_frame) if rig else model_from_scene(sub, sub_index)
        keep_img = keep_frame[img_frame] | (rig and cid.max(initial=-1) == -1)
        images = {int(i): model[1][int(i)] for i in img_ids[keep_img]}
        write_model(path, model[0], images, *model[2:], fmt=fmt)
        written.append(path)
    return written


# ---------------------------------------------------------------------------- command line
def _main(argv=None):
    """``python -m glomap_b200.colmap_io to-flat MODEL_DIR FLAT.bin`` converts a COLMAP sparse model into the flat
    binary problem of ``b200sfm_cli ba|gp`` (trivial frames);
    ``from-flat MODEL_DIR FLAT.bin OUT_DIR`` writes the solved state back as a COLMAP model;
    ``prune MODEL_DIR OUT_DIR [--min_num_observations N]`` splits a model into its covisibility clusters on the GPU
    (PruneWeaklyConnectedImages, the ``mapper_resume --skip_pruning 0`` analogue for trivial frames) and writes one model
    per cluster to OUT_DIR/0, OUT_DIR/1, ...  Every subcommand reads camera models 0-3 (SIMPLE_PINHOLE, PINHOLE,
    SIMPLE_RADIAL, RADIAL) only: the flat problem holds those, and ``prune`` recomputes the points' reprojection errors of
    the models it writes.  The pruning itself does not read the intrinsics.  ``glomap_b200.mapper_resume`` runs the
    global mapper on a model, rigs included."""
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
