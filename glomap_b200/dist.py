"""Host-side plumbing for the one-process-per-GPU layout (torch.distributed is
used only for rendezvous: the NCCL unique id broadcast, barriers, and the
max-over-ranks timing; the data-path all-reduces run inside libb200sfm.so).

Sharding contract (SURVEY.md 8(e)): points -- with all their observations --
are partitioned across ranks in contiguous chunk ranges; cameras and intrinsics
are replicated; every rank calls the solver collectively.
"""
from __future__ import annotations

import os

import numpy as np


def env_rank_world():
    return int(os.environ.get("RANK", "0")), int(os.environ.get("WORLD_SIZE", "1")), int(os.environ.get("LOCAL_RANK", "0"))


def shard_range(n_items: int, chunk: int, rank: int, world: int) -> tuple[int, int]:
    """Contiguous, chunk-aligned range of items owned by ``rank``."""
    nchunks = (n_items + chunk - 1) // chunk
    a = (nchunks * rank) // world
    b = (nchunks * (rank + 1)) // world
    return a * chunk, min(n_items, b * chunk)


def shard_scene(scene, rank: int, world: int, chunk: int = 1):
    """Slice a full flat scene into the shard of ``rank`` (points
    [a, b) and their observations); cameras/intrinsics are replicated.  The shard owns COPIES of every array a
    solver updates in place (poses, points, intrinsics): solving a shard never touches ``scene``."""
    from .synthetic import RigScene, Scene
    a, b = shard_range(scene.P, chunk, rank, world)
    o0, o1 = int(scene.pt_obs_begin[a]), int(scene.pt_obs_begin[b])
    if isinstance(scene, RigScene):   # known rigs: frames, sensors, intrinsics and the rig layout are replicated
        return RigScene(scene.quat.copy(), scene.trans.copy(), scene.points[a:b].copy(),
                        (scene.pt_obs_begin[a:b + 1] - o0).astype(np.int64), scene.obs_frame[o0:o1], scene.obs_sensor[o0:o1],
                        scene.obs_xy[o0:o1], scene.sensor_quat.copy(), scene.sensor_trans.copy(), scene.sensor_intr,
                        scene.intr_model, scene.intr_params.copy(), scene.image_frame, scene.image_sensor, scene.frame_rig,
                        scene.sensor_rig, scene.rig_ref_sensor, scene.sensor_known), (a, b)
    return Scene(scene.quat.copy(), scene.trans.copy(), scene.points[a:b].copy(), (scene.pt_obs_begin[a:b + 1] - o0).astype(np.int64),
                 scene.obs_cam[o0:o1], scene.obs_xy[o0:o1], scene.cam_intr, scene.intr_model, scene.intr_params.copy()), (a, b)


def broadcast_nccl_id(make_id, rank: int, world: int) -> bytes | None:
    """Rank 0 creates the id (b200sfm_nccl_unique_id), everyone receives it
    through the already-initialised torch.distributed default group."""
    if world == 1:
        return None
    import torch.distributed as dist
    obj = [make_id() if rank == 0 else None]
    dist.broadcast_object_list(obj, src=0)
    return obj[0]
