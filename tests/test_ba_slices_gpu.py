"""The bundle adjuster's camera-order rows grouped by point slice (DESIGN.md §3), forced with B200SFM_PT_SLICES on
scenes whose per-point records fit L2 and would otherwise keep one slice (the plain camera order):
  * the first LM step of the stored-row intrinsics path (nk = 1) against the FP64 sparse reference, through the
    operator-level probe and bounds of test_ba_system_gpu.py, on a scene that reaches the shapes the slicing creates;
  * a whole solve against the C oracle at a tight PCG tolerance (same LM iteration count);
  * the sharded solve against the single-GPU one, when two GPUs are visible."""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import test_ba_gpu as TB  # noqa: E402
import test_ba_system_gpu as TS  # noqa: E402
import test_multigpu_gpu as TM  # noqa: E402
from test_ba_system_gpu import scenes  # noqa: E402,F401  (module-scoped scene cache, a fixture)
from glomap_b200 import estimators as E, synthetic as S  # noqa: E402
from oracle import ba_oracle as B, ba_oracle_fast as F  # noqa: E402

pytestmark = pytest.mark.gpu

# two slices of 2048 points (whole ELL windows) on the P = 2600 scene of test_ba_system_gpu.py, the last one partial
SLICED = "ell_pt_slices_kfast_nk1_K200"
SLICED_PATH = (dict(K=200), dict(optimize_intrinsics=True), {"B200SFM_PT_SLICES": "2"}, dict(use_ell=1, kfast=1, nk=1))


def test_sliced_scene_reaches_its_shapes(scenes):
    """The (slice, camera) buckets include one of more than 256 observations (several segments) and a camera with
    observations in one slice and none in the other.  Three slices would be 1024 points wide, and none of their
    buckets passes 256."""
    sc = scenes(SLICED_PATH[0])
    lens = np.diff(sc.pt_obs_begin)
    used = np.repeat(lens >= TS.MIN_VIEWS, lens)
    n = np.zeros((2, sc.C), int)
    np.add.at(n, (np.repeat(np.arange(sc.P), lens)[used] // 2048, sc.obs_cam[used]), 1)
    assert sc.P % 2048 != 0 and n.max() > 256 and ((n == 0) & (n.sum(0) > 0)).any()


def test_sliced_device_step_matches_the_fp64_reference(scenes, monkeypatch):
    monkeypatch.setitem(TS.PATHS, SLICED, SLICED_PATH)
    TS.test_device_step_matches_the_fp64_reference(SLICED, scenes, monkeypatch)


def test_point_sliced_camera_order_tracks_the_oracle(monkeypatch):
    """Three slices of 1024 points, the last one partial: same trajectory as the C oracle."""
    monkeypatch.setenv("B200SFM_PT_SLICES", "3")
    sc = S.make_scene(60, 3000, mean_track_len=7, seed=17, pixel_sigma=0.5)
    init = S.perturb_scene(sc)
    mask = E.first_frame_mask(sc.C)
    ok, dev, st = TB._device_solve(init, mask, tol=1e-12)
    x, summ = F.solve_ba_fast(*TB._oracle_args(sc, init), B.BAOptions(), mask)
    assert ok and st.iterations == summ.iterations
    assert abs(st.final_cost - summ.final_cost) <= 1e-8 * summ.final_cost
    rot, cen = TB._compare(dev, x)
    assert rot < 1e-4 and cen < 1e-6


def test_sharded_ba_with_point_slices_matches_single_gpu(monkeypatch):
    """tests/multigpu_ba_check.py with the rows grouped by point slice on every rank and in the single-GPU solve."""
    n = TM._ngpu()
    if n < 2:
        pytest.skip(f"needs 2 GPUs on one box, {n} visible (NCCL ranks cannot share a device)")
    monkeypatch.setenv("B200SFM_PT_SLICES", "3")
    out = TM._run("multigpu_ba_check.py", 2, 29521)
    assert "multi-GPU parity OK" in out, out[-2000:]
