"""The per-segment epilogues of the camera-order kernels (ba2_linearize_cams, ba2_pass_b, ba2_schur_diag): the warp
reduce-scatter of the segment sums, one atomic per lane that holds a total, and the lane-parallel B^T M B of a known
rig's Schur-Jacobi block.

test_ba_system_gpu.py and test_ba_pass_b_rounds_gpu.py compare these kernels with the FP64 reference on trivial
frames, known rigs and two intrinsics parameters per camera (NK = 2: the 27 frame sums and the 17 intrinsics sums
take two reduce-scatter rounds).  What they do not build:
  * a known rig whose frames have constant rotation or translation, so the lane-parallel conjugation and the masked
    rows and columns of the Schur-Jacobi block meet, against the FP64 reference;
  * bit-identical U, g_c, the Schur-Jacobi preconditioner, the right-hand side and the mat-vec over two runs when
    every camera is one segment, with NK = 0 and NK = 2: each address then takes one atomic, so the per-segment sums
    themselves must be reproducible.
"""
import numpy as np
import pytest

import test_ba_system_gpu as T
from glomap_b200 import estimators as E, synthetic as S

pytestmark = pytest.mark.gpu

RIG_MASKS = {3: 1, 4: 2, 5: 3}   # frames of the rig scene with constant rotation / translation / both


def test_known_rig_schur_jacobi_with_masked_frames_matches_the_fp64_reference():
    sc = T.make_rig(model=S.SIMPLE_PINHOLE)
    mask = E.first_frame_mask(sc.C)
    for f, m in RIG_MASKS.items():
        mask[f] = m
    probe = T.Probe(sc, {}, mask)
    out, dev = probe.step(T.LOOSE_K)
    assert out.use_ell == 1 and out.ext == 0
    ref = probe.oracle(out.nbk, T.expected_precond(probe, out))
    err = dict(U=T.blockerr(dev["U"], T.BS.pack_sym(ref.U_blocks), 21), g_c=T.blockerr(dev["g_c"], ref.g_c, 6),
               b=T.blockerr(dev["b"], ref.b, 6), Minv=T.blockerr(dev["Minv"], T.BS.pack_sym(ref.Minv_blocks), 21))
    rng = np.random.default_rng(5)
    x = np.where(ref.var_c, rng.normal(size=ref.var_c.size), 0.0)
    err["apply"] = T.blockerr(probe.apply(x), ref.apply(x), 6)
    print("rig_masked", " ".join(f"{k}={v:.1e}" for k, v in err.items()))
    assert not {k: v for k, v in err.items() if not v <= T.BOUNDS[k]}, err


@pytest.mark.parametrize("model,nk", [(S.SIMPLE_PINHOLE, 0), (S.PINHOLE, 2)])
def test_one_segment_per_camera_is_bit_identical_across_runs(model, nk, monkeypatch):
    monkeypatch.setenv("B200SFM_PT_SLICES", "1")
    C = 40
    sc = S.make_scene(C, 800, mean_track_len=6, seed=3, pixel_sigma=0.8, model=model, num_intrinsics=C)
    sc = S.perturb_scene(sc, rot_deg=0.05, center_frac=0.001, point_frac=0.001, seed=3)
    lens = np.diff(sc.pt_obs_begin)
    used = np.bincount(sc.obs_cam[np.repeat(lens >= T.MIN_VIEWS, lens)], minlength=C)
    assert used.max() < 256 + 128   # one camera-order segment per camera (seg_split)
    mask = E.first_frame_mask(C)
    mask[1], mask[2] = 1, 2
    x = np.random.default_rng(9).normal(size=(C + C) * 6)
    runs = []
    for _ in range(2):
        probe = T.Probe(sc, dict(optimize_intrinsics=nk > 0), mask)
        out, dev = probe.step(3)
        assert out.nk == nk and out.use_ell == 1
        xv = np.where(dev["jscale_c"] < 0, 0.0, x[:out.nbk * 6])
        runs.append((dev, probe.apply(xv)))
    (d0, y0), (d1, y1) = runs
    for f in ("U", "g_c", "Minv", "b", "px"):
        assert np.array_equal(d0[f], d1[f]), f
    assert np.array_equal(y0, y1)
    assert np.abs(y0).max() > 0 and np.abs(d0["U"]).max() > 0
