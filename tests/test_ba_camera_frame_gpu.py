"""Operator-level tests of the camera-frame camera-order kernels (pass B, the Schur-Jacobi diagonal, the camera-order
linearisation) and of the pinhole form of the projection, against the FP64 sparse reference, through the probe and
the bounds of test_ba_system_gpu.py.

The cases are the ones that file does not build: constant intrinsics on the v2 / ELL path with PINHOLE (fx != fy),
SIMPLE_RADIAL and RADIAL; a scene whose intrinsics blocks mix k = 0 (pinhole form) and k != 0 (radial form), so both
projection branches run in one launch and inside one point-order warp; known rigs on SIMPLE_PINHOLE; and the
camera-order rows grouped in two point slices.
"""
import numpy as np
import pytest

import test_ba_system_gpu as T
from glomap_b200 import synthetic as S

pytestmark = pytest.mark.gpu
_make_intrinsics = S.make_intrinsics


def _mixed_k_intrinsics(*args, **kwargs):
    """SIMPLE_RADIAL blocks with k = 0 on every other block: neighbouring cameras (cam_intr = c % K) take different
    projection branches."""
    cam_intr, intr_model, intr_params = _make_intrinsics(*args, **kwargs)
    intr_params = intr_params.copy()
    intr_params[::2, 3] = 0.0
    return cam_intr, intr_model, intr_params


PATHS = {
    "ell_pinhole_K1": (dict(K=1, model=S.PINHOLE), {}, {}, dict(use_v2=1, use_ell=1, ext=0)),
    "ell_simple_radial_K3": (dict(K=3, model=S.SIMPLE_RADIAL), {}, {}, dict(use_v2=1, use_ell=1, ext=0)),
    "ell_radial_K1": (dict(K=1, model=S.RADIAL), {}, {}, dict(use_v2=1, use_ell=1, ext=0)),
    "ell_mixed_k_K8": ("mixed", {}, {}, dict(use_v2=1, use_ell=1, ext=0)),
    "kfast_mixed_k_K8": ("mixed", dict(optimize_intrinsics=True), {}, dict(use_ell=1, kfast=1, nk=2)),
    "rig_known_simple_pinhole": ("rig_pinhole", {}, {}, dict(use_ell=1, ext=0)),
    "ell_slices2_K1": (dict(K=1), {}, {"B200SFM_PT_SLICES": "2"}, dict(use_v2=1, use_ell=1, ext=0)),
}


def _scene(spec, monkeypatch):
    if spec == "mixed":
        with monkeypatch.context() as m:
            m.setattr(S, "make_intrinsics", _mixed_k_intrinsics)
            sc = T.make_scene(K=8, model=S.SIMPLE_RADIAL)
        k = sc.intr_params[:, 3]
        assert (k == 0).any() and (k != 0).any()
        return sc
    if spec == "rig_pinhole":
        return T.make_rig(model=S.SIMPLE_PINHOLE)
    return T.make_scene(**spec)


@pytest.mark.parametrize("name", list(PATHS))
def test_camera_frame_step_matches_the_fp64_reference(name, monkeypatch):
    spec, opts, env, want = PATHS[name]
    sc = _scene(spec, monkeypatch)
    # reuse the whole comparison of test_ba_system_gpu.py: its scene cache is bypassed with this case's scene
    monkeypatch.setitem(T.PATHS, name, ("rig" if spec == "rig_pinhole" else {}, opts, env, want))
    T.test_device_step_matches_the_fp64_reference(name, lambda _spec: sc, monkeypatch)
