"""``SolveRotationAveraging`` (glomap/controllers/rotation_averager.cc:8-63,183-197), the driver of
``glomap rotation_averager``: gravity-aligned, stratified rotation averaging over ``estimators.RotationEstimator``.

With gravity and ``use_stratified`` the pairs whose two frames have gravity are solved first as a 1-DoF problem on their
largest component, unless there is no such pair or they are more than 95 % of all pairs; the whole graph is then solved
starting from that result.  Frames are the view graph's nodes (trivial rigs; for known rigs pass the frame graph of
``estimators.rig_view_graph``).  The pre-pass for cameras with an unknown cam_from_rig (.cc:65-182) is not restated."""
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


def _estimate_on(mask, vg, options, R0, gravity, ctx):
    """EstimateRotations over the nodes of ``mask`` and the pairs between them (nodes renumbered in ascending order)."""
    from .synthetic import ViewGraph
    idx = np.nonzero(mask)[0]
    remap = np.full(vg.n_images, -1, np.int64)
    remap[idx] = np.arange(len(idx))
    ei, ej = np.asarray(vg.ei), np.asarray(vg.ej)
    k = mask[ei] & mask[ej]
    sub = ViewGraph(len(idx), remap[ei[k]].astype(np.int32), remap[ej[k]].astype(np.int32), np.asarray(vg.R_rel)[k],
                    np.asarray(vg.weight)[k], np.asarray(vg.R_gt)[idx])
    ok, R = RotationEstimator(options, ctx).EstimateRotations(sub, R0[idx], gravity=None if gravity is None else gravity[idx])
    return ok, idx, R


def solve_rotation_averaging(vg, gravity=None, options: RotationAveragerOptions | None = None, R_init=None, ctx=None):
    """``gravity`` [n,3] with NaN rows for frames without a prior (None: no gravity); ``R_init`` [n,3,3] the initial
    rotations (``ReadGravity`` sets R_align for the frames with gravity, the identity elsewhere).  Returns
    (ok, R [n,3,3] (R_init outside the solved component), registered [n] bool)."""
    o = options or RotationAveragerOptions()
    n = vg.n_images
    R = np.tile(np.eye(3), (n, 1, 1)) if R_init is None else np.array(R_init, dtype=np.float64, copy=True)
    g = None if gravity is None else np.asarray(gravity, dtype=np.float64)
    has = np.zeros(n, bool) if g is None else ~np.isnan(g).any(axis=1)
    ei, ej = np.asarray(vg.ei), np.asarray(vg.ej)
    reg = largest_component(n, ei, ej)                                           # .cc:13
    grav_pair = reg[ei] & reg[ej] & has[ei] & has[ej]
    solve_1dof = o.use_gravity and o.use_stratified and g is not None and stratified_branch(vg, g, reg)
    est_opts = RotationEstimatorOptions(**{f.name: getattr(o, f.name) for f in dataclasses.fields(RotationEstimatorOptions)})
    if solve_1dof:
        sub = _subgraph(vg, grav_pair)
        mask = largest_component(n, sub.ei, sub.ej, reg)                          # .cc:56
        ok, idx, R_sub = _estimate_on(mask, sub, est_opts, R, g, ctx)            # .cc:57-61
        if not ok:
            return False, R, mask
        R[idx] = R_sub
    ok, idx, R_all = _estimate_on(reg, vg, est_opts, R, g if o.use_gravity else None, ctx)   # .cc:184-195
    if R_all is not None:
        R[idx] = R_all
    return ok, R, reg


def stratified_branch(vg, gravity, registered=None) -> bool:
    """Whether SolveRotationAveraging solves the 1-DoF subsystem first (.cc:42-50), given gravity and use_stratified."""
    g = np.asarray(gravity, dtype=np.float64)
    has = ~np.isnan(g).any(axis=1)
    ei, ej = np.asarray(vg.ei), np.asarray(vg.ej)
    reg = largest_component(vg.n_images, ei, ej) if registered is None else np.asarray(registered, bool)
    pair_in = reg[ei] & reg[ej]
    grav_pairs = int((pair_in & has[ei] & has[ej]).sum())
    return not (grav_pairs == 0 or grav_pairs > int(pair_in.sum()) * 0.95)
