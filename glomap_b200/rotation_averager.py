"""``SolveRotationAveraging`` (glomap/controllers/rotation_averager.cc:8-63,183-197), the driver of
``glomap rotation_averager``: gravity-aligned, stratified rotation averaging over ``estimators.RotationEstimator``.

With gravity and ``use_stratified`` the pairs whose two frames have gravity are solved first as a 1-DoF problem on their
largest component, unless there is no such pair or they are more than 95 % of all pairs; the whole graph is then solved
starting from that result.  Frames are the view graph's nodes (trivial rigs; for known rigs pass the frame graph of
``estimators.rig_view_graph``).

``solve_rotation_averaging_rig`` is the same driver for rigs given image by image.  When a camera's cam_from_rig is not
known yet it runs the reference's pre-pass (.cc:65-182): a rotation averaging in which every image of such a camera is a
frame of its own, whose result ``ConvertRotationsFromImageToRig`` turns into first cam_from_rig and rig_from_world
rotations (rotation_initializer.py, on the device) before the real solve starts from them.  With gravity every
cam_from_rig must be known, as in the reference: the image pairs are folded onto the frames and the frame graph goes
through the gravity-aligned, stratified driver above."""
from __future__ import annotations

import dataclasses

import numpy as np

from .estimators import RotationEstimator, RotationEstimatorOptions


@dataclasses.dataclass
class RotationAveragerOptions(RotationEstimatorOptions):
    """controllers/rotation_averager.h:7-12."""
    use_stratified: bool = True


def largest_component(n: int, ei, ej, registered=None) -> np.ndarray:
    """KeepLargestConnectedComponents (scene/view_graph.cc:56-97) over the pairs whose two nodes are ``registered``:
    the mask of the nodes of the largest component (the one with the smallest node among equally large ones); all
    False without a pair."""
    import scipy.sparse as sp
    from scipy.sparse.csgraph import connected_components
    ei, ej = np.asarray(ei, np.int64), np.asarray(ej, np.int64)
    reg = np.ones(n, bool) if registered is None else np.asarray(registered, bool)
    k = reg[ei] & reg[ej]
    if not k.any():
        return np.zeros(n, bool)
    G = sp.coo_matrix((np.ones(int(k.sum())), (ei[k], ej[k])), shape=(n, n))
    _, lab = connected_components(G, directed=False)
    in_edge = np.zeros(n, bool)
    in_edge[ei[k]] = in_edge[ej[k]] = True
    sizes = np.bincount(lab[in_edge], minlength=lab.max() + 1)
    return in_edge & (lab == int(np.argmax(sizes)))


def _subgraph(vg, keep_edge):
    from .synthetic import ViewGraph
    return ViewGraph(vg.n_images, np.asarray(vg.ei)[keep_edge], np.asarray(vg.ej)[keep_edge], np.asarray(vg.R_rel)[keep_edge],
                     np.asarray(vg.weight)[keep_edge], vg.R_gt)


def _estimate_on(mask, vg, R0, gravity, estimate):
    """``estimate`` over the nodes of ``mask`` and the pairs between them (nodes renumbered in ascending order)."""
    from .synthetic import ViewGraph
    idx = np.nonzero(mask)[0]
    remap = np.full(vg.n_images, -1, np.int64)
    remap[idx] = np.arange(len(idx))
    ei, ej = np.asarray(vg.ei), np.asarray(vg.ej)
    k = mask[ei] & mask[ej]
    sub = ViewGraph(len(idx), remap[ei[k]].astype(np.int32), remap[ej[k]].astype(np.int32), np.asarray(vg.R_rel)[k],
                    np.asarray(vg.weight)[k], None if vg.R_gt is None else np.asarray(vg.R_gt)[idx])
    ok, R = estimate(sub, R0[idx], None if gravity is None else gravity[idx])
    return ok, idx, R


def _estimator_options(o: RotationAveragerOptions) -> RotationEstimatorOptions:
    return RotationEstimatorOptions(**{f.name: getattr(o, f.name) for f in dataclasses.fields(RotationEstimatorOptions)})


def _solve_frames(vg, g, o, R, estimate, solve_1dof, info):
    """.cc:13-63,183-197 over the frame graph ``vg``: the 1-DoF pass over the largest component of the pairs whose two
    frames have gravity when ``solve_1dof``, then the whole largest component from its result.  ``estimate(vg, R0,
    gravity)`` -> (ok, R) is RotationEstimator::EstimateRotations."""
    n = vg.n_images
    has = np.zeros(n, bool) if g is None else ~np.isnan(g).any(axis=1)
    ei, ej = np.asarray(vg.ei), np.asarray(vg.ej)
    reg = largest_component(n, ei, ej)                                           # .cc:13
    grav_pair = reg[ei] & reg[ej] & has[ei] & has[ej]
    if solve_1dof is None:
        if g is not None:
            info["gravity_pairs"], info["total_pairs"] = _count_gravity_pairs(ei, ej, reg, has)
        solve_1dof = o.use_gravity and o.use_stratified and g is not None and _stratify(info["gravity_pairs"], info["total_pairs"])
    info["stratified"] = bool(solve_1dof)
    if solve_1dof:
        sub = _subgraph(vg, grav_pair)
        mask = largest_component(n, sub.ei, sub.ej, reg)                          # .cc:56
        ok, idx, R_sub = _estimate_on(mask, sub, R, g, estimate)                  # .cc:57-61
        if not ok:
            return False, R, mask
        R[idx] = R_sub
    ok, idx, R_all = _estimate_on(reg, vg, R, g if o.use_gravity else None, estimate)   # .cc:184-195
    if R_all is not None:
        R[idx] = R_all
    return ok, R, reg


def solve_rotation_averaging(vg, gravity=None, options: RotationAveragerOptions | None = None, R_init=None, ctx=None,
                             info=None):
    """``gravity`` [n,3] with NaN rows for frames without a prior (None: no gravity); ``R_init`` [n,3,3] the initial
    rotations (``ReadGravity`` sets R_align for the frames with gravity, the identity elsewhere).  Returns
    (ok, R [n,3,3] (R_init outside the solved component), registered [n] bool).  ``info``, when a dict, receives
    ``gravity_pairs`` / ``total_pairs`` (the pairs of the largest component with gravity at both ends / all of them) and
    ``stratified`` (whether the 1-DoF pass ran)."""
    o = options or RotationAveragerOptions()
    n = vg.n_images
    R = np.tile(np.eye(3), (n, 1, 1)) if R_init is None else np.array(R_init, dtype=np.float64, copy=True)
    g = None if gravity is None else np.asarray(gravity, dtype=np.float64)
    est_opts = _estimator_options(o)
    info = {} if info is None else info

    def estimate(sub, R0, grav):
        return RotationEstimator(est_opts, ctx).EstimateRotations(sub, R0, gravity=grav)

    return _solve_frames(vg, g, o, R, estimate, None, info)


def _count_gravity_pairs(ei, ej, registered, has_gravity):
    """(pairs between registered nodes whose two nodes have gravity, pairs between registered nodes) (.cc:22-40)."""
    ei, ej = np.asarray(ei), np.asarray(ej)
    pair_in = registered[ei] & registered[ej]
    return int((pair_in & has_gravity[ei] & has_gravity[ej]).sum()), int(pair_in.sum())


def stratified_branch(vg, gravity, registered=None) -> bool:
    """Whether SolveRotationAveraging solves the 1-DoF subsystem first (.cc:42-50), given gravity and use_stratified."""
    g = np.asarray(gravity, dtype=np.float64)
    has = ~np.isnan(g).any(axis=1)
    reg = largest_component(vg.n_images, vg.ei, vg.ej) if registered is None else np.asarray(registered, bool)
    return _stratify(*_count_gravity_pairs(vg.ei, vg.ej, reg, has))


def _stratify(grav_pairs: int, total_pairs: int) -> bool:
    """.cc:49-50: no 1-DoF pass without a gravity pair or with more than 95 % of the pairs gravity pairs."""
    return not (grav_pairs == 0 or grav_pairs > total_pairs * 0.95)


# ---------------------------------------------------------------------------
# Rigs, image by image (SolveRotationAveraging .cc:8-197 without gravity)
# ---------------------------------------------------------------------------
def _sub_view_graph(vg, node_of_image, n_nodes, keep_edge):
    """The pairs ``keep_edge`` with their images renumbered by ``node_of_image`` (every kept image has a node)."""
    from .synthetic import ViewGraph
    ei, ej = np.asarray(vg.ei)[keep_edge], np.asarray(vg.ej)[keep_edge]
    return ViewGraph(n_nodes, node_of_image[ei].astype(np.int32), node_of_image[ej].astype(np.int32),
                     np.asarray(vg.R_rel)[keep_edge], np.asarray(vg.weight)[keep_edge], np.tile(np.eye(3), (n_nodes, 1, 1)))


def trivial_layout(image_frame, image_camera, camera_known, frame_ref_camera, image_registered):
    """The trivial rigs of the pre-pass (.cc:84-158): frame f < F keeps its registered images of known cameras, and every
    registered image of an unknown camera becomes a frame F + k of its own (k in ascending image order), whose reference
    camera is that camera.  Returns (trivial frame [I] (-1: not registered), reference camera [F + #own frames])."""
    fr = np.asarray(image_frame, np.int64)
    cam = np.asarray(image_camera, np.int64)
    reg = np.asarray(image_registered, bool)
    own = reg & ~np.asarray(camera_known, bool)[cam]
    F = len(frame_ref_camera)
    tf = np.where(reg, fr, -1)
    tf[own] = F + np.arange(int(own.sum()))
    return tf, np.concatenate([np.asarray(frame_ref_camera, np.int64), cam[own]])


def fold_pairs(vg, node_of_image, R_cam_from_rig, image_camera):
    """Image pairs onto frames with the known cam_from_rig rotations (global_rotation_averaging.cc:274-309):
    R_rel = R_c2^T R_21 R_c1 for the pairs whose two images have a node; pairs inside one node are dropped (.cc:300-303).
    Returns (keep [E] bool, ei, ej, R_rel)."""
    ei, ej = np.asarray(vg.ei), np.asarray(vg.ej)
    ni, nj = node_of_image[ei], node_of_image[ej]
    keep = (ni >= 0) & (nj >= 0) & (ni != nj)
    cam = np.asarray(image_camera)
    R1, R2 = R_cam_from_rig[cam[ei[keep]]], R_cam_from_rig[cam[ej[keep]]]
    R = np.einsum("nji,njk,nkl->nil", R2, np.asarray(vg.R_rel)[keep], R1)
    return keep, ni[keep], nj[keep], R


class _DeviceOps:
    """The numeric steps of solve_rotation_averaging_rig on the device; oracle/rig_init_oracle.py supplies numpy ones."""

    def __init__(self, options: RotationEstimatorOptions, ctx):
        from .estimators import default_context
        self.options, self.ctx = options, ctx or default_context()

    def mst(self, vg):
        """InitializeFromMaximumSpanningTree's tree and composition (root: node 0).  Returns (R [n,3,3], reached [n])."""
        from .estimators import initialize_from_maximum_spanning_tree_device
        R, parent = initialize_from_maximum_spanning_tree_device(vg, None, self.ctx, root=0)
        return R, parent >= 0

    def convert(self, *args, **kw):
        from .rotation_initializer import convert_rotations_from_image_to_rig
        return convert_rotations_from_image_to_rig(*args, ctx=self.ctx, **kw)

    def estimate(self, vg, R0):
        """RotationEstimator with skip_initialization over a frame graph.  Returns (ok, R, (l1, irls) iterations)."""
        est = RotationEstimator(dataclasses.replace(self.options, skip_initialization=True), self.ctx)
        ok, R = est.EstimateRotations(vg, R0)
        return ok, R, (est.summary.l1_iterations, est.summary.irls_iterations)

    def estimate_gravity(self, vg, R0, gravity):
        """RotationEstimator with use_gravity over a frame graph: the frames with a prior (non-NaN rows of ``gravity``)
        are 1-DoF.  Returns (ok, R)."""
        return RotationEstimator(self.options, self.ctx).EstimateRotations(vg, R0, gravity=gravity)

    def estimate_rig(self, g, R_frames0, R_cams0):
        """RotationEstimator with unknown cam_from_rig rotations over rig_view_graph_unknown's layout."""
        from .estimators import estimate_rotations_rig_unknown
        est = RotationEstimator(dataclasses.replace(self.options, skip_initialization=True), self.ctx)
        ok, Rf, Rc = estimate_rotations_rig_unknown(est, g, R_frames0, R_cams0)
        return ok, Rf, Rc, (est.summary.l1_iterations, est.summary.irls_iterations)


def _image_rotations(vg, image_mask, ops):
    """Image-level maximum spanning tree over the pairs between the images of ``image_mask``, rooted at the first of them
    (the shim's smallest id).  Returns (R [I,3,3], reached [I])."""
    I = len(image_mask)
    node = np.full(I, -1, np.int64)
    idx = np.nonzero(image_mask)[0]
    node[idx] = np.arange(len(idx))
    R = np.tile(np.eye(3), (I, 1, 1))
    reached = np.zeros(I, bool)
    if len(idx) == 0:
        return R, reached
    ei, ej = np.asarray(vg.ei), np.asarray(vg.ej)
    Rs, rs = ops.mst(_sub_view_graph(vg, node, len(idx), image_mask[ei] & image_mask[ej]))
    R[idx], reached[idx] = Rs, rs
    return R, reached


def image_has_gravity(image_frame, image_camera, frame_ref_camera, camera_known, frame_gravity):
    """Image::HasGravity (scene/image.h:78-84): the image's frame has a prior (a non-NaN row of ``frame_gravity`` [F,3])
    and its camera is the frame's reference camera or has a known cam_from_rig.  Returns [I] bool."""
    fr, cam = np.asarray(image_frame, np.int64), np.asarray(image_camera, np.int64)
    has_frame = ~np.isnan(np.asarray(frame_gravity, np.float64)).any(axis=1)
    return has_frame[fr] & ((cam == np.asarray(frame_ref_camera, np.int64)[fr]) | np.asarray(camera_known, bool)[cam])


def _solve_rig_gravity(vg, fr, cam, known, R_cam, ref_cam, gravity, o, R, reg, ops, info):
    """.cc:13-63,183-197 with use_gravity and every cam_from_rig known: the image pairs folded onto the frames with the
    known rotations (self loops dropped), then the frame-graph driver with the frames' priors.  The 1-DoF pass is chosen
    on the image pairs, as the reference counts them (.cc:22-50)."""
    from .synthetic import ViewGraph
    F = len(ref_cam)
    ei, ej = np.asarray(vg.ei), np.asarray(vg.ej)
    img_g = image_has_gravity(fr, cam, ref_cam, known, gravity)
    pair_in = reg[fr[ei]] & reg[fr[ej]]
    n_grav, n_total = int((pair_in & img_g[ei] & img_g[ej]).sum()), int(pair_in.sum())
    info["gravity_pairs"], info["total_pairs"] = n_grav, n_total
    solve_1dof = o.use_stratified and _stratify(n_grav, n_total)
    keep, fi, fj, R_rel = fold_pairs(vg, fr, R_cam, cam)
    fg = ViewGraph(F, fi.astype(np.int32), fj.astype(np.int32), R_rel, np.asarray(vg.weight)[keep], np.tile(np.eye(3), (F, 1, 1)))
    ok, R, mask = _solve_frames(fg, gravity, o, R, ops.estimate_gravity, solve_1dof, info)
    return ok, R, R_cam, mask


def _solve_rig(vg, image_frame, image_camera, camera_known, cam_from_rig, frame_ref_camera, o, R_init, ops, info,
               gravity=None):
    from . import geometry as geo
    from .estimators import rig_view_graph, rig_view_graph_unknown
    fr = np.asarray(image_frame, np.int64)
    cam = np.asarray(image_camera, np.int64)
    ref_cam = np.asarray(frame_ref_camera, np.int64)
    F, K, I = len(ref_cam), len(camera_known), len(fr)
    known = np.array(camera_known, dtype=bool, copy=True)
    known[ref_cam] = True
    q_cam = np.array(np.reshape(cam_from_rig, (K, 4)), dtype=np.float64, copy=True)
    q_cam[ref_cam] = [0.0, 0.0, 0.0, 1.0]
    R_cam = geo.quat_xyzw_to_rotmat(q_cam)
    R = np.tile(np.eye(3), (F, 1, 1)) if R_init is None else np.array(R_init, dtype=np.float64, copy=True)
    ei, ej = np.asarray(vg.ei), np.asarray(vg.ej)
    reg = largest_component(F, fr[ei], fr[ej])                                    # .cc:13
    unknown = ~known
    if o.use_gravity and unknown.any():                                           # global_rotation_averaging.cc:47-59
        info.setdefault("log", []).append(
            f"rotation averaging: use_gravity needs every cam_from_rig, camera(s) {np.flatnonzero(unknown).tolist()} "
            "have none")
        return False, R, R_cam, reg
    if o.use_gravity and gravity is not None:
        return _solve_rig_gravity(vg, fr, cam, known, R_cam, ref_cam, np.asarray(gravity, np.float64), o, R, reg, ops, info)
    img_reg = reg[fr]
    pair_ok = np.ones(len(ei), bool)
    cam_init = np.zeros(K, bool)                                                  # unknown cameras with an average
    if unknown.any() and not o.skip_initialization:
        # ---- the pre-pass (.cc:81-175) ----
        tf, tref = trivial_layout(fr, cam, known, ref_cam, img_reg)
        nT = len(tref)
        R_triv = R_cam.copy()
        R_triv[unknown] = np.eye(3)                                               # the reference sensor of its own rig
        keep, ti, tj, TR = fold_pairs(vg, tf, R_triv, cam)
        tmask = largest_component(nT, ti, tj)                                     # .cc:160
        img_t = (tf >= 0) & tmask[np.maximum(tf, 0)]
        pair_ok = img_t[ei] & img_t[ej]                                           # the pairs that stay valid
        R_img, reached = _image_rotations(vg, img_t, ops)                         # InitializeFromMaximumSpanningTree
        q_triv = geo.rotmat_to_quat_xyzw_fast(R_triv)
        _, _, fq, _ = ops.convert(np.where(img_t, tf, -1), cam, geo.rotmat_to_quat_xyzw_fast(R_img), tref, np.ones(K, np.uint8),
                                  q_triv, np.tile([0.0, 0.0, 0.0, 1.0], (nT, 1)), image_estimated=reached)
        tnode = np.full(nT, -1, np.int64)
        tidx = np.nonzero(tmask)[0]
        tnode[tidx] = np.arange(len(tidx))
        k = tmask[ti] & tmask[tj]
        from .synthetic import ViewGraph
        tvg = ViewGraph(len(tidx), tnode[ti[k]].astype(np.int32), tnode[tj[k]].astype(np.int32), TR[k],
                        np.asarray(vg.weight)[keep][k], np.tile(np.eye(3), (len(tidx), 1, 1)))
        ok_t, R_t, its = ops.estimate(tvg, geo.quat_xyzw_to_rotmat(fq[tidx]))    # .cc:162-166
        info["trivial"] = its
        R_tf = np.tile(np.eye(3), (nT, 1, 1))
        if ok_t:
            R_tf[tidx] = R_t
        R_img = np.einsum("nij,njk->nik", R_triv[cam], R_tf[np.maximum(tf, 0)])   # cam_from_world of the images (.cc:169-173)
        est = img_t if ok_t else np.zeros(I, bool)
    else:
        # ---- .cc:183-196: the initialisation is forced on when a camera is unknown; its images are skipped ----
        if o.skip_initialization and not unknown.any():
            R_img, est = None, None
        else:
            R_img, reached = _image_rotations(vg, img_reg, ops)
            est = reached & known[cam]
    fn = None
    if R_img is not None:                                                         # ConvertRotationsFromImageToRig (.cc:175)
        cq, cn, fq, fn = ops.convert(np.where(img_reg, fr, -1), cam, geo.rotmat_to_quat_xyzw_fast(R_img), ref_cam,
                                     known.astype(np.uint8), q_cam, geo.rotmat_to_quat_xyzw_fast(R), image_estimated=est)
        cam_init = unknown & (cn > 0)
        R_cam[cam_init] = geo.quat_xyzw_to_rotmat(cq[cam_init])
        R[fn > 0] = geo.quat_xyzw_to_rotmat(fq[fn > 0])
    # ---- the solve from those rotations (.cc:177-182 / 192-195) over the frames of the remaining pairs ----
    mask = largest_component(F, fr[ei[pair_ok]], fr[ej[pair_ok]], reg)
    if not mask.any():
        return False, R, R_cam, mask
    fnode = np.full(F, -1, np.int64)
    fidx = np.nonzero(mask)[0]
    fnode[fidx] = np.arange(len(fidx))
    img_in = mask[fr]
    inode = np.full(I, -1, np.int64)
    iidx = np.nonzero(img_in)[0]
    inode[iidx] = np.arange(len(iidx))
    svg = _sub_view_graph(vg, inode, len(iidx), pair_ok & img_in[ei] & img_in[ej])
    sf, sc = fnode[fr[iidx]], cam[iidx]
    seen = np.zeros(K, bool)
    seen[sc] = True
    solve_unknown = unknown & seen
    q_known = geo.rotmat_to_quat_xyzw_fast(R_cam)
    if solve_unknown.any():
        g = rig_view_graph_unknown(svg, sf, sc, q_known, ~solve_unknown)
        ucams = np.nonzero(solve_unknown)[0]
        ok, Rf, Rc, its = ops.estimate_rig(g, R[fidx], np.where(cam_init[ucams][:, None, None], R_cam[ucams], np.eye(3)))
        if ok:
            R_cam[ucams] = Rc
    else:
        fg = rig_view_graph(svg, sf, sc, q_known)
        ok, Rf, its = ops.estimate(fg, R[fidx])
    info["final"] = its
    if Rf is not None:
        R[fidx] = Rf
    return ok, R, R_cam, mask


def solve_rotation_averaging_rig(vg, image_frame, image_camera, camera_known, cam_from_rig, frame_ref_camera,
                                 options: RotationAveragerOptions | None = None, R_init=None, ctx=None, info=None,
                                 gravity=None):
    """SolveRotationAveraging (.cc:8-197) for rigs.

    ``vg``: the image-level view graph (cam2_from_cam1 per pair); image_frame [I] and image_camera [I]: every image's
    frame and camera; camera_known [K] and cam_from_rig [K,4] (xyzw): the cameras whose cam_from_rig is known and those
    rotations (the reference camera of each frame is known, with the identity); frame_ref_camera [F]; R_init [F,3,3]:
    rig_from_world rotations to start from where the initialisation leaves a frame without a sample (identity without).

    With an unknown camera and not skip_initialization, the pre-pass runs (.cc:81-182): the trivial rigs of
    ``trivial_layout``, their pairs folded with the known cam_from_rig and restricted to their largest component, the
    image-level maximum spanning tree, ConvertRotationsFromImageToRig for the trivial rigs, a rotation averaging of the
    trivial frames, the image rotations composed from it and ConvertRotationsFromImageToRig for the real rigs; the
    solve with the unknown cam_from_rig rotations then starts from those averages (global_rotation_averaging.cc:183-188).
    Pairs with an image outside the trivial largest component leave the view graph, as in the reference.  Otherwise
    (.cc:183-196) the initialisation is forced on when a camera is unknown: images of unknown cameras are skipped and
    those cameras start from zero (global_rotation_averaging.cc:239-242).  The solve runs over the largest component of
    the remaining pairs.

    ``gravity`` [F,3]: one prior per frame (NaN rows: none), read only with use_gravity.  With use_gravity and a camera
    whose cam_from_rig is not known the call returns False (.cc:47-59) before any solve, and says why in
    ``info["log"]``.  With every cam_from_rig known and ``gravity``, the image pairs are folded onto the frames
    (global_rotation_averaging.cc:274-309, pairs inside one frame dropped) and aligned with their frames' R_align
    (.cc:311-326); the frames with a prior are 1-DoF, the first of them is the gauge (.cc:207-217); with use_stratified
    the pairs whose two images have gravity (``image_has_gravity``) are solved first on their largest component unless
    there is none or they are more than 95 % of the pairs (rotation_averager.cc:15-63), and the whole graph then starts
    from that result.  This is ``solve_rotation_averaging`` on the frame graph of ``estimators.rig_view_graph``, except
    that the 95 % rule counts image pairs, pairs inside one frame included, as the reference does.

    Returns (ok, R [F,3,3] rig_from_world rotations (R_init outside the solved frames), R_cam [K,3,3] cam_from_rig
    rotations (the estimates for the unknown cameras with images; known ones unchanged), registered [F] bool).  ``info``,
    when a dict, receives the (L1, IRLS) iteration counts of the trivial and the final solve; with gravity,
    ``gravity_pairs`` / ``total_pairs`` / ``stratified``."""
    o = options or RotationAveragerOptions()
    return _solve_rig(vg, image_frame, image_camera, camera_known, cam_from_rig, frame_ref_camera, o, R_init,
                      _DeviceOps(_estimator_options(o), ctx), {} if info is None else info, gravity)
