"""The view-graph passes of stage 3 on the GPU (b200sfm_view_graph_filter_rotations / _keep_largest_component,
view_graph_kernels.cuh) against the host restatements of glomap_b200/view_graph.py, bit for bit: seeded random graphs
with multi-image frames, outlier pairs and several components, the 100 000-frame lattice, bad indices, and the mapper end
to end with images outside the largest component."""
import ctypes as ct

import numpy as np
import pytest

from glomap_b200 import _lib, estimators as E, geometry as G, mapper as M, synthetic as S, view_graph as VG

pytestmark = pytest.mark.gpu


def _random_graph(rng, F, per_frame, E_, comps, outlier):
    """Frames split into ``comps`` blocks (pairs only inside a block); images of a frame share its rotation up to a
    per-image offset; ``outlier`` of the pairs carry a random rotation."""
    image_frame = np.repeat(np.arange(F), rng.integers(1, per_frame + 1, size=F)).astype(np.int32)
    I = len(image_frame)
    block = rng.integers(0, comps, size=F)
    a = rng.integers(0, I, size=E_)
    by_block = [np.flatnonzero(block[image_frame] == c) for c in range(comps)]
    b = np.array([rng.choice(by_block[block[image_frame[x]]]) for x in a])
    R = G.so3_exp(rng.normal(size=(I, 3)))
    Rr = G.so3_exp(rng.normal(size=(E_, 3)) * np.radians(2.0)) @ R[b] @ np.swapaxes(R[a], -1, -2)
    out = rng.uniform(size=E_) < outlier
    Rr[out] = G.so3_exp(rng.normal(size=(int(out.sum()), 3)))
    q, qr = G.rotmat_to_quat_xyzw_fast(R), G.rotmat_to_quat_xyzw_fast(Rr)
    return image_frame, a.astype(np.int32), b.astype(np.int32), q, qr


@pytest.mark.parametrize("seed", range(8))
def test_device_equals_host_on_random_graphs(seed):
    rng = np.random.default_rng(seed)
    F = int(rng.integers(20, 400))
    image_frame, a, b, q, qr = _random_graph(rng, F, 3, int(rng.integers(300, 3000)), int(rng.integers(1, 5)),
                                             [0.01, 0.05, 0.1, 0.3][seed % 4])
    I, E_ = len(image_frame), len(a)
    valid0 = rng.uniform(size=E_) > 0.05
    img_reg = rng.uniform(size=I) > 0.05
    thr = float(rng.uniform(3, 20))
    vh, nh = VG.filter_rotations(q, a, b, qr, thr, valid0, img_reg)
    vd, nd = VG.filter_rotations_device(q, a, b, qr, thr, valid0, img_reg)
    assert np.array_equal(vh, vd) and nh == nd
    freg0 = rng.uniform(size=F) > 0.1
    h = VG.keep_largest_connected_components(F, image_frame, a, b, vh, freg0)
    d = VG.keep_largest_connected_components_device(F, image_frame, a, b, vd, freg0)
    assert np.array_equal(h[0], d[0]) and np.array_equal(h[1], d[1]) and h[2] == d[2] and h[2] > 0
    # repeated calls give the same result
    d2 = VG.keep_largest_connected_components_device(F, image_frame, a, b, vd, freg0)
    assert np.array_equal(d[0], d2[0]) and np.array_equal(d[1], d2[1]) and d[2] == d2[2]


def test_ties_self_loops_and_no_valid_pair_on_the_device():
    # two equally large components {4, 5} and {1, 3}, a self-loop frame 0 (images 0, 6)
    image_frame = np.array([0, 1, 2, 3, 4, 5, 0], np.int32)
    a, b = np.array([4, 3, 0], np.int32), np.array([5, 1, 6], np.int32)
    for valid in ([True, True, True], [True, True, False], [False, False, False]):
        reg0 = np.array([1, 0, 1, 0, 1, 1], bool)
        h = VG.keep_largest_connected_components(6, image_frame, a, b, valid, reg0)
        d = VG.keep_largest_connected_components_device(6, image_frame, a, b, valid, reg0)
        assert np.array_equal(h[0], d[0]) and np.array_equal(h[1], d[1]) and h[2] == d[2]
    assert d[2] == 0 and d[1].tolist() == reg0.tolist()
    # the angle at the threshold and NaN keep the pair
    q = np.array([[0, 0, 0, 1], [0, 0, np.sin(0.1), np.cos(0.1)], [np.nan, 0, 0, 1]])
    qr = np.array([[0, 0, 0, 1.0], [0, 0, 0, 1.0]])
    ang = VG.rotation_angle_deg(tuple(q[1]), tuple(qr[0]))
    for thr in (ang, np.nextafter(ang, 0), np.nextafter(ang, 90)):
        h = VG.filter_rotations(q, [0, 0], [1, 2], qr, thr)
        d = VG.filter_rotations_device(q, [0, 0], [1, 2], qr, thr)
        assert h[0].tolist() == d[0].tolist() and h[1] == d[1]
        assert d[0][1]


def test_lattice_100k_frames_5m_pairs():
    vg = S.make_lattice_view_graph(100_000, 100, seed=1, noise_deg=2.0, outlier_ratio=0.05)
    side = int(np.ceil(np.sqrt(vg.n_images)))
    q, qr = G.rotmat_to_quat_xyzw_fast(vg.R_gt), G.rotmat_to_quat_xyzw_fast(vg.R_rel)
    # cut the lattice in two: no valid pair crosses row 10
    valid0 = (vg.ei // side < 10) == (vg.ej // side < 10)
    vh, nh = VG.filter_rotations(q, vg.ei, vg.ej, qr, 10.0, valid0)
    vd, nd = VG.filter_rotations_device(q, vg.ei, vg.ej, qr, 10.0, valid0)
    assert np.array_equal(vh, vd) and nh == nd and nh > 0.04 * vg.E
    frame = np.arange(vg.n_images, dtype=np.int32)
    h = VG.keep_largest_connected_components(vg.n_images, frame, vg.ei, vg.ej, vh)
    d = VG.keep_largest_connected_components_device(vg.n_images, frame, vg.ei, vg.ej, vd)
    assert np.array_equal(h[0], d[0]) and np.array_equal(h[1], d[1]) and h[2] == d[2]
    assert d[2] == vg.n_images - 10 * side


def test_bad_indices_are_refused_without_touching_the_outputs():
    ctx = E.default_context()
    q = np.array([[0, 0, 0, 1.0]] * 3)
    qr = np.array([[0, 0, 0.5, 0.5]] * 2)
    for a, b in (([0, 3], [1, 2]), ([0, -1], [1, 2]), ([0, 1], [2, 1 << 20])):
        with pytest.raises(_lib.B200Error) as ei:
            VG.filter_rotations_device(q, a, b, qr, 1.0, ctx=ctx)
        assert ei.value.code == 1
        with pytest.raises(_lib.B200Error) as ei:
            VG.keep_largest_connected_components_device(3, [0, 1, 2], a, b, ctx=ctx)
        assert ei.value.code == 1
    with pytest.raises(_lib.B200Error):                    # an image's frame outside [0, F)
        VG.keep_largest_connected_components_device(3, [0, 3, 2], [0], [1], ctx=ctx)
    # outputs untouched on refusal
    lib = ctx.lib
    valid = np.array([1, 1], np.uint8)
    reg = np.array([1, 0, 1], np.uint8)
    i1, i2, fr = np.array([0, 5], np.int32), np.array([1, 2], np.int32), np.array([0, 1, 2], np.int32)
    n32 = ct.c_int32(-1)
    p = lambda x: x.ctypes.data_as(ct.c_void_p)   # noqa: E731
    assert lib.b200sfm_view_graph_keep_largest_component(ctx.handle, 3, 3, p(fr), 2, p(i1), p(i2), p(valid), p(reg),
                                                         ct.byref(n32)) == 1
    assert valid.tolist() == [1, 1] and reg.tolist() == [1, 0, 1]
    # the context still works
    out = VG.filter_rotations_device(q, [0, 1], [1, 2], qr, 1.0, ctx=ctx)
    assert out[1] == 2 and not out[0].any()


# ---- mapper end to end ------------------------------------------------------------------------------------------------
class _Recording:
    """Wraps a solver class and records (number of cameras, observations) of every problem it is given."""
    seen = []

    @classmethod
    def wrap(cls, base):
        class W(base):
            def Solve(self, prob, *args, **kw):
                cls.seen.append((len(prob.quat), np.asarray(prob.obs_xy if hasattr(prob, "obs_xy") else prob.bearings).copy()))
                return super().Solve(prob, *args, **kw)
        return W


def test_mapper_drops_the_images_outside_the_largest_component(monkeypatch):
    sc = S.make_scene(30, 3000, mean_track_len=6, seed=21, pixel_sigma=0.5)
    vg = S.view_graph_from_scene(sc, min_shared=8, noise_deg=0.5)
    rng = np.random.default_rng(7)
    cut = np.array([3, 11, 20])
    # every pair of the three images carries a rotation error of 40-90 degrees.  A robust rotation average fits an
    # image to at least one of its pairs, so that alone leaves each of them attached; their pairs to the other images are
    # therefore dropped, and the three form a component of their own, outside the largest one.
    hit = np.isin(vg.ei, cut) | np.isin(vg.ej, cut)
    inside = np.isin(vg.ei, cut) & np.isin(vg.ej, cut)
    w = rng.normal(size=(int(hit.sum()), 3))
    w /= np.linalg.norm(w, axis=1, keepdims=True)
    w *= np.radians(rng.uniform(40, 90, size=(len(w), 1)))
    vg.R_rel[hit] = G.so3_exp(w) @ vg.R_rel[hit]
    keep = ~hit | inside
    vg = S.ViewGraph(vg.n_images, vg.ei[keep], vg.ej[keep], vg.R_rel[keep], vg.weight[keep], vg.R_gt)
    assert vg.E >= M.VIEW_GRAPH_DEVICE_MIN_PAIRS                 # the passes run on the device
    start = sc.copy()
    start.quat[:] = [0, 0, 0, 1]
    start.trans[:] = np.arange(sc.C)[:, None] * [1.0, 2.0, 3.0]
    start.points[:] = 0
    _Recording.seen = []
    monkeypatch.setattr(M.E, "GlobalPositioner", _Recording.wrap(E.GlobalPositioner))
    monkeypatch.setattr(M.E, "BundleAdjuster", _Recording.wrap(E.BundleAdjuster))
    opts = M.GlobalMapperOptions()
    opts.opt_ba.optimize_intrinsics = False
    mapper = M.GlobalMapper(opts)
    ok, out = mapper.Solve(vg, start)
    assert ok, mapper.log
    assert np.flatnonzero(~mapper.image_registered).tolist() == cut.tolist(), mapper.log
    reg = mapper.image_registered
    # unregistered cameras keep their input pose and no observation of theirs is left
    assert np.array_equal(out.quat[cut], start.quat[cut]) and np.array_equal(out.trans[cut], start.trans[cut])
    assert not np.isin(out.obs_cam, cut).any()
    # no observation of an unregistered image reached global positioning or bundle adjustment
    assert len(_Recording.seen) >= 3
    assert all(C == int(reg.sum()) for C, _ in _Recording.seen)  # the problems hold the registered cameras only
    cut_xy = {tuple(r) for r in sc.obs_xy[np.isin(sc.obs_cam, cut)]}
    for _, arr in _Recording.seen[1:]:                           # bundle adjustment: pixel observations
        assert not any(tuple(r) in cut_xy for r in np.asarray(arr).reshape(-1, 2))
    n_reg_obs = int(np.isin(sc.obs_cam, np.flatnonzero(reg)).sum())
    assert len(_Recording.seen[0][1]) <= n_reg_obs               # global positioning: one bearing per kept observation
    # registered poses: the reference's noisy thresholds after Sim3 alignment (global_mapper_test.cc:213-215)
    rot, cen = G.compare_reconstructions(G.quat_xyzw_to_rotmat(out.quat[reg]), out.trans[reg],
                                         G.quat_xyzw_to_rotmat(sc.quat[reg]), sc.trans[reg])[:2]
    assert rot < 1e-1 and cen < 1e-1, (rot, cen, mapper.log)
