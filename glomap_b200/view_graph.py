"""The two view-graph passes ``GlobalMapper::Solve`` runs after each rotation averaging (glomap/controllers/
global_mapper.cc:91-115), on flat arrays:

* ``filter_rotations`` = ``RelPoseFilter::FilterRotations`` (processors/relpose_filter.cc:7-33): a valid pair whose two
  images are registered is invalidated when the angle between ``q2 * q1^-1`` (the images' cam_from_world rotations) and
  its cam2_from_cam1 rotation is larger than ``max_angle_deg``.  The angle is Eigen's ``angularDistance`` (the Rigid3d
  overload of ``CalcAngle``, math/rigid3d.cc:7-9); an angle equal to the threshold, or NaN, keeps the pair.
* ``keep_largest_connected_components`` = ``ViewGraph::KeepLargestConnectedComponents`` (scene/view_graph.cc:56-97) in
  frame space: the frames of the valid pairs are the nodes; the largest component stays registered (ties: the component
  holding the smallest frame index), every other frame is deregistered and every pair with an image outside it
  invalidated; returns the number of registered images.  Without a valid pair nothing changes and 0 is returned.

Both are host restatements written as loops in the reference's form; they are what the device versions
(``*_device``, through ``b200sfm_view_graph_filter_rotations`` / ``b200sfm_view_graph_keep_largest_component``,
view_graph_kernels.cuh) are tested against.  Quaternions are xyzw.  The rules for ties, NaN and the empty graph are the
ones include/b200sfm.h states."""
from __future__ import annotations

import ctypes as ct
import math
from collections import deque

import numpy as np


def _qmul(a, b):
    """Eigen's quat_product (xyzw), in its term order."""
    ax, ay, az, aw = a
    bx, by, bz, bw = b
    return (aw * bx + ax * bw + ay * bz - az * by,
            aw * by + ay * bw + az * bx - ax * bz,
            aw * bz + az * bw + ax * by - ay * bx,
            aw * bw - ax * bx - ay * by - az * bz)


def rotation_angle_deg(q_calc, q_rel) -> float:
    """``CalcAngle(Rigid3d, Rigid3d)``: q_calc.angularDistance(q_rel) in degrees, 2 atan2(|d.vec|, |d.w|) with
    d = q_calc * conj(q_rel)."""
    dx, dy, dz, dw = _qmul(q_calc, (-q_rel[0], -q_rel[1], -q_rel[2], q_rel[3]))
    return 2.0 * math.atan2(math.sqrt(dx * dx + dy * dy + dz * dz), abs(dw)) * 180.0 / math.pi


def filter_rotations(cam_from_world_quat, pair_image1, pair_image2, pair_quat, max_angle_deg: float, pair_valid=None,
                     image_registered=None):
    """Returns (pair_valid [E] bool, number of pairs invalidated).  ``cam_from_world_quat`` [I,4] per image,
    ``pair_quat`` [E,4] cam2_from_cam1 per pair; ``pair_valid`` / ``image_registered`` default to all True.
    ``Inverse`` and the normalisation of Rigid3d's product only scale a quaternion by a positive factor, which the angle
    does not depend on: the conjugate stands for the inverse and the product is not normalised (as on the device)."""
    q = np.asarray(cam_from_world_quat, np.float64).reshape(-1, 4).tolist()
    qr = np.asarray(pair_quat, np.float64).reshape(-1, 4).tolist()
    i1, i2 = np.asarray(pair_image1).tolist(), np.asarray(pair_image2).tolist()
    valid = np.ones(len(i1), bool) if pair_valid is None else np.array(pair_valid, bool)
    reg = None if image_registered is None else np.asarray(image_registered, bool).tolist()
    num_invalid = 0
    for e in range(len(i1)):
        if not valid[e]:
            continue
        a, b = i1[e], i2[e]
        if reg is not None and (not reg[a] or not reg[b]):
            continue
        qa = q[a]
        q_calc = _qmul(q[b], (-qa[0], -qa[1], -qa[2], qa[3]))   # image2.CamFromWorld() * Inverse(image1.CamFromWorld())
        if rotation_angle_deg(q_calc, qr[e]) > max_angle_deg:
            valid[e] = False
            num_invalid += 1
    return valid, num_invalid


def keep_largest_connected_components(num_frames: int, image_frame, pair_image1, pair_image2, pair_valid=None,
                                      frame_registered=None):
    """Returns (pair_valid [E] bool, frame_registered [F] bool, number of registered images).  ``image_frame`` [I] is
    the frame of every image; ``frame_registered`` (default all True) is returned unchanged without a valid pair."""
    F = int(num_frames)
    img_frame = np.asarray(image_frame).tolist()
    i1, i2 = np.asarray(pair_image1).tolist(), np.asarray(pair_image2).tolist()
    valid = np.ones(len(i1), bool) if pair_valid is None else np.array(pair_valid, bool)
    reg = np.ones(F, bool) if frame_registered is None else np.array(frame_registered, bool)
    adjacency: dict[int, set] = {}                                          # CreateFrameAdjacencyList (:140-150)
    for e in range(len(i1)):
        if valid[e]:
            f1, f2 = img_frame[i1[e]], img_frame[i2[e]]
            adjacency.setdefault(f1, set()).add(f2)
            adjacency.setdefault(f2, set()).add(f1)
    visited, components = set(), []                                        # FindConnectedComponents (:33-52)
    for root in sorted(adjacency):
        if root in visited:
            continue
        comp, queue = {root}, deque([root])
        visited.add(root)
        while queue:
            cur = queue.popleft()
            for nb in adjacency[cur]:
                if nb not in visited:
                    visited.add(nb)
                    comp.add(nb)
                    queue.append(nb)
        components.append(comp)
    best, max_img = None, 0                                                 # :62-69, ties to the smallest frame
    for comp in components:                                                 # (components come in ascending smallest frame)
        if len(comp) > max_img:
            best, max_img = comp, len(comp)
    if max_img == 0:
        return valid, reg, 0
    reg[:] = False                                                          # :76-83
    for f in best:
        reg[f] = True
    for e in range(len(i1)):                                                # :84-90
        if not reg[img_frame[i1[e]]] or not reg[img_frame[i2[e]]]:
            valid[e] = False
    return valid, reg, sum(1 for f in img_frame if reg[f])                  # :92-96


# ---- device -----------------------------------------------------------------------------------------------------------
def _ptr(a):
    return a.ctypes.data_as(ct.c_void_p) if a is not None and a.size else None


def _index_array(a, name):
    from .reconstruction_pruning import _as_int_array
    return _as_int_array(a, np.int32, name)


def filter_rotations_device(cam_from_world_quat, pair_image1, pair_image2, pair_quat, max_angle_deg: float, pair_valid=None,
                            image_registered=None, ctx=None):
    """``filter_rotations`` on the GPU; same arguments and return value."""
    from . import _lib, estimators as E
    q = np.ascontiguousarray(np.asarray(cam_from_world_quat, np.float64).reshape(-1, 4))
    i1, i2 = _index_array(pair_image1, "pair_image1"), _index_array(pair_image2, "pair_image2")
    qr = np.ascontiguousarray(np.asarray(pair_quat, np.float64).reshape(-1, 4))
    E_ = len(i1)
    if len(i2) != E_ or len(qr) != E_:
        raise ValueError("pair_image1, pair_image2 and pair_quat must have one entry per pair")
    valid = np.ones(E_, np.uint8) if pair_valid is None else np.ascontiguousarray(np.asarray(pair_valid, bool).astype(np.uint8))
    reg = None if image_registered is None else np.ascontiguousarray(np.asarray(image_registered, bool).astype(np.uint8))
    if valid.shape != (E_,) or (reg is not None and reg.shape != (len(q),)):
        raise ValueError("pair_valid must have one entry per pair and image_registered one per image")
    ctx = ctx or E.default_context()
    n = ct.c_int64(0)
    _lib.check(ctx.handle, ctx.lib.b200sfm_view_graph_filter_rotations(
        ctx.handle, len(q), _ptr(q), _ptr(reg), E_, _ptr(i1), _ptr(i2), _ptr(qr), float(max_angle_deg), _ptr(valid),
        ct.byref(n)))
    return valid.astype(bool), int(n.value)


def keep_largest_connected_components_device(num_frames: int, image_frame, pair_image1, pair_image2, pair_valid=None,
                                             frame_registered=None, ctx=None):
    """``keep_largest_connected_components`` on the GPU; same arguments and return value."""
    from . import _lib, estimators as E
    F = int(num_frames)
    fr = _index_array(image_frame, "image_frame")
    i1, i2 = _index_array(pair_image1, "pair_image1"), _index_array(pair_image2, "pair_image2")
    E_ = len(i1)
    if len(i2) != E_:
        raise ValueError("pair_image1 and pair_image2 must have one entry per pair")
    valid = np.ones(E_, np.uint8) if pair_valid is None else np.ascontiguousarray(np.asarray(pair_valid, bool).astype(np.uint8))
    reg = np.ones(F, np.uint8) if frame_registered is None else np.ascontiguousarray(np.asarray(frame_registered, bool).astype(np.uint8))
    if valid.shape != (E_,) or reg.shape != (F,):
        raise ValueError("pair_valid must have one entry per pair and frame_registered one per frame")
    ctx = ctx or E.default_context()
    n = ct.c_int32(0)
    _lib.check(ctx.handle, ctx.lib.b200sfm_view_graph_keep_largest_component(
        ctx.handle, F, len(fr), _ptr(fr), E_, _ptr(i1), _ptr(i2), _ptr(valid), _ptr(reg), ct.byref(n)))
    return valid.astype(bool), reg.astype(bool), int(n.value)
