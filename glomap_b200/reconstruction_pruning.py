"""Reconstruction pruning (stage 8 of ``GlobalMapper::Solve``, glomap/controllers/global_mapper.cc:340-353, on with
``--skip_pruning 0``) on the GPU: ``prune_weakly_connected_images`` = PruneWeaklyConnectedImages
(glomap/processors/reconstruction_pruning.cc:6-131) through ``b200sfm_prune_weakly_connected`` (prune_kernels.cuh).

The frames are split into covisibility clusters: frame pairs seen together by >= 5 observation pairs of the tracks longer
than 2 form a weighted visibility graph; its largest component is kept (``is_registered``) and cut into clusters joined
by strong edges (weight > max(median - MAD, 20)) or by >= 2 slightly weaker ones (EstablishStrongClusters).  Clusters
are numbered by size, descending; ``colmap_io.write_clustered_model`` writes one model per cluster.

For a trivial-frame ``synthetic.Scene`` the inputs are ``scene.pt_obs_begin``, ``scene.obs_cam`` and ``scene.C``.  The CPU
restatement is oracle/pruning_oracle.py; ties and the empty case follow the rules of include/b200sfm.h."""
from __future__ import annotations

import ctypes as ct

import numpy as np


def prune_weakly_connected_images(track_begin, obs_frame, num_frames: int, frame_self_loop=None, min_num_observations: int = 0,
                                  ctx=None, is_registered=None, max_pair_keys_per_pass: int = 0) -> dict:
    """Tracks as a CSR (``track_begin`` [T+1]) over the frame index of every observation (``obs_frame``, 0..F-1);
    ``frame_self_loop`` [F] marks frames with >= 2 images present (rigs; None for trivial frames).  ``is_registered``
    [F] is the registration before the call (default: all registered); it is returned unchanged when there is no
    visibility edge.  Returns dict(cluster_id [F] int32 (-1 outside every cluster), is_registered [F] bool,
    num_clusters, stats (dict of b200sfm_prune_stats))."""
    from . import _lib, estimators as E_
    F = int(num_frames)
    tb = _as_int_array(track_begin, np.int64, "track_begin")
    if tb.size == 0:
        tb = np.zeros(1, np.int64)
    of = _as_int_array(obs_frame, np.int32, "obs_frame")
    if tb.ndim != 1 or of.ndim != 1:
        raise ValueError("track_begin and obs_frame must be 1-D")
    if len(of) != tb[-1]:
        raise ValueError(f"obs_frame has {len(of)} entries, track_begin[-1] = {int(tb[-1])}")
    loop = None if frame_self_loop is None else np.ascontiguousarray(np.asarray(frame_self_loop, np.uint8))
    reg = np.ones(F, np.uint8) if is_registered is None else np.ascontiguousarray(np.asarray(is_registered, np.uint8).copy())
    for name, a in (("frame_self_loop", loop), ("is_registered", reg)):
        if a is not None and a.shape != (F,):
            raise ValueError(f"{name} must have num_frames = {F} entries, not {a.shape}")
    ctx = ctx or E_.default_context()
    cid = np.full(F, -1, np.int32)
    nc = ct.c_int32(0)
    st = _lib.PruneStats()
    ptr = lambda a: a.ctypes.data_as(ct.c_void_p) if a is not None and a.size else None   # noqa: E731
    _lib.check(ctx.handle, ctx.lib.b200sfm_prune_weakly_connected(
        ctx.handle, F, len(tb) - 1, ptr(tb), ptr(of), ptr(loop), int(min_num_observations), int(max_pair_keys_per_pass),
        ptr(cid), ptr(reg), ct.byref(nc), ct.byref(st)))
    return dict(cluster_id=cid, is_registered=reg.astype(bool), num_clusters=int(nc.value), stats=st.as_dict())


def _as_int_array(a, dtype, name):
    """Contiguous array of ``dtype``; integers that do not fit it raise instead of wrapping (an index of 2^31 would wrap
    into [0, F) and pass the device's range check)."""
    a = np.asarray(a)
    if a.size == 0:
        return np.zeros(a.shape, dtype)
    if a.dtype.kind not in "iu":
        raise ValueError(f"{name} must be an integer array, not {a.dtype}")
    info = np.iinfo(dtype)
    if not np.can_cast(a.dtype, dtype, "safe") and (a.min() < info.min or a.max() > info.max):   # only where it can wrap
        raise ValueError(f"{name} has entries outside the range of {np.dtype(dtype).name}")
    return np.ascontiguousarray(a.astype(dtype, copy=False))
