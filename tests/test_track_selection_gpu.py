"""Device track selection (b200sfm_tracks_select, TrackEngine::FindTracksForProblem) against the host loop and the literal
transcription of tests/test_track_selection_cpu.py: index work, so every comparison is exact.  Also the shim's TrackEngine
built against the library, and mapper stage 4."""
import importlib.util
import os
import subprocess

import numpy as np
import pytest

from glomap_b200 import _lib, mapper as MP, synthetic as S, track_establishment as TE

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)


def _load(name):
    spec = importlib.util.spec_from_file_location("_" + name, os.path.join(HERE, name + ".py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


_sel_cpu = _load("test_track_selection_cpu")
_te_cpu = _load("test_track_establishment_cpu")


def _same(a: TE.Tracks, b: TE.Tracks):
    assert np.array_equal(a.track_ids, b.track_ids)
    assert np.array_equal(a.begin, b.begin)
    assert np.array_equal(a.obs_image, b.obs_image) and np.array_equal(a.obs_feature, b.obs_feature)


def _mask(tracks, selected: TE.Tracks):
    return _sel_cpu.mask_of(tracks, selected.track_ids)


@pytest.mark.parametrize("drop", [0.0, 0.3])
@pytest.mark.parametrize("quota", [-1, 0, 1, 5])
def test_device_selection_equals_the_host_on_establishment_scenes(drop, quota):
    """The scenes of test_tracks_gpu.py, with some images unregistered."""
    sc = S.make_scene(40, 4000, mean_track_len=6, seed=71)
    features, pairs = _te_cpu._pairs_from_scene(sc, np.random.default_rng(5), drop)[:2]
    full, _ = TE.establish_full_tracks_device(pairs, features)
    for registered in (range(1, sc.C + 1), range(1, sc.C + 1, 3)):
        o = TE.TrackEstablishmentOptions(min_num_tracks_per_view=quota)
        _same(TE.find_tracks_for_problem_device(full, registered, o), TE.find_tracks_for_problem(full, registered, o))


@pytest.mark.parametrize("seed", range(40))
def test_device_selection_equals_the_host_on_random_track_sets(seed):
    """Unsorted observations, repeated images, ties in length, quotas -5..5, caps 0 / 1 / 5 / 50, no registered image."""
    rng = np.random.default_rng(seed)
    tracks, registered = _sel_cpu.random_tracks(rng, T=int(rng.integers(1, 3000)), I=int(rng.integers(1, 60)))
    for k in range(6):
        o = _sel_cpu.random_options(rng)
        reg = registered if k < 5 else []
        want = TE.find_tracks_for_problem(tracks, reg, o)
        got = TE.find_tracks_for_problem_device(tracks, reg, o)
        _same(got, want)
        assert _mask(tracks, got).tolist() == _sel_cpu.parallel_select(tracks, reg, o).tolist()


@pytest.mark.parametrize("field,value", [("min_num_view_per_track", -1), ("max_num_view_per_track", -1),
                                         ("max_num_tracks", -1), ("max_num_tracks", -7)])
def test_negative_options_follow_the_reference(field, value):
    for seed in range(8):
        rng = np.random.default_rng(500 + seed)
        tracks, registered = _sel_cpu.random_tracks(rng, T=int(rng.integers(1, 2000)), I=30, max_len=14)
        o = _sel_cpu.random_options(rng)
        setattr(o, field, value)
        ref = _sel_cpu.reference_select(_sel_cpu.as_dict(tracks), registered, o)
        got = TE.find_tracks_for_problem_device(tracks, registered, o)
        assert _sel_cpu.as_dict(got) == ref
        assert got.track_ids.tolist() == sorted(ref, key=lambda t: (len(_sel_cpu.as_dict(tracks)[t]), t), reverse=True)


def test_long_tracks_and_caps():
    """Tracks far longer than a warp, max_num_view_per_track < 0, and a cap that bites without a quota."""
    rng = np.random.default_rng(9)
    tracks, registered = _sel_cpu.random_tracks(rng, T=300, I=40, max_len=600)
    for o in (TE.TrackEstablishmentOptions(max_num_view_per_track=-1, max_num_tracks=17),
              TE.TrackEstablishmentOptions(max_num_view_per_track=-1, min_num_tracks_per_view=3),
              TE.TrackEstablishmentOptions(max_num_view_per_track=1000, max_num_tracks=0)):
        ref = _sel_cpu.reference_select(_sel_cpu.as_dict(tracks), registered, o)
        assert _sel_cpu.as_dict(TE.find_tracks_for_problem_device(tracks, registered, o)) == ref
    assert len(TE.find_tracks_for_problem_device(tracks, registered, TE.TrackEstablishmentOptions(max_num_tracks=0))) == 1


def test_empty_and_invalid_inputs():
    empty = TE.Tracks(np.zeros(0, np.uint64), np.zeros(1, np.int64), np.zeros(0, np.uint32), np.zeros(0, np.uint32))
    got = TE.find_tracks_for_problem_device(empty, [1, 2])
    assert len(got) == 0 and got.begin.tolist() == [0]
    dup = TE.Tracks(np.array([5, 9, 5], np.uint64), np.array([0, 3, 6, 9]), np.array([1, 2, 3] * 3, np.uint32), np.zeros(9, np.uint32))
    with pytest.raises(_lib.B200Error) as e:
        TE.find_tracks_for_problem_device(dup, [1, 2, 3])
    assert e.value.code == 1 and "track id" in str(e.value)
    bad = TE.Tracks(np.array([5, 9], np.uint64), np.array([0, 4, 3]), np.array([1, 2, 3], np.uint32), np.zeros(3, np.uint32))
    with pytest.raises(_lib.B200Error) as e:
        TE.find_tracks_for_problem_device(bad, [1, 2, 3])
    assert e.value.code == 1 and "non-decreasing" in str(e.value)
    # the context stays usable after the refusals
    ok = TE.Tracks(np.array([5, 9], np.uint64), np.array([0, 3, 6]), np.array([1, 2, 3] * 2, np.uint32), np.zeros(6, np.uint32))
    assert TE.find_tracks_for_problem_device(ok, [1, 2, 3]).track_ids.tolist() == [9, 5]


def _write_world(path, features, pairs, registered, o):
    lines = [f"images {len(features)}"]
    for i in sorted(features):
        xy = np.asarray(features[i], np.float64)
        lines.append(f"{i} {int(i in registered)} {len(xy)} " + " ".join(repr(float(v)) for v in xy.ravel()))
    lines.append(f"pairs {len(pairs)}")
    for p in pairs:
        m = np.asarray(p.matches)
        lines.append(f"{p.image_id1} {p.image_id2} {int(p.is_valid)} {len(m)} " + " ".join(str(int(v)) for v in m.ravel())
                     + f" {len(p.inliers)} " + " ".join(str(int(v)) for v in p.inliers))
    lines.append(f"options {o.min_num_tracks_per_view} {o.min_num_view_per_track} {o.max_num_view_per_track} {o.max_num_tracks} "
                 f"{o.thres_inconsistency!r}")
    path.write_text("\n".join(lines) + "\n")


def _print(what, tracks: TE.Tracks):
    out = [f"{what} {len(tracks)}"]
    for t in np.argsort(tracks.track_ids, kind="stable"):
        im, ft = tracks.observations(int(t))
        tid = int(tracks.track_ids[t])
        out.append(f"track {tid} {tid}" + "".join(f" {int(a)}:{int(b)}" for a, b in zip(im, ft)))
    return out


@pytest.mark.parametrize("quota", [-1, 2])
def test_shim_track_engine_reproduces_the_python_result(tmp_path, quota):
    sc = S.make_scene(20, 1500, mean_track_len=5, seed=73)
    rng = np.random.default_rng(8)
    features, pairs = _te_cpu._pairs_from_scene(sc, rng, 0.2)[:2]
    for p in pairs[::5]:                                    # wrong matches: some tracks are discarded
        m = np.array(p.matches)
        m[:3, 1] = rng.permutation(m[:, 1])[:3]
        p.matches = m
    pairs[2].is_valid = False
    registered = set(range(1, sc.C + 1)) - {4, 11}
    o = TE.TrackEstablishmentOptions(min_num_tracks_per_view=quota, max_num_tracks=400)
    full, dis = TE.establish_full_tracks_device(pairs, features, o)
    assert dis > 0
    sel = TE.find_tracks_for_problem_device(full, sorted(registered), o)
    world = tmp_path / "world.txt"
    _write_world(world, features, pairs, registered, o)
    exe = tmp_path / "track_driver"
    libdir = os.path.join(ROOT, "glomap_b200")
    subprocess.run(["g++", "-std=c++17", "-O1", "-Wall", "-Werror", "-I" + os.path.join(ROOT, "glomap_b200", "host"), "-o", str(exe),
                    os.path.join(HERE, "shim_mock", "track_driver.cc"), "-L" + libdir, "-lb200sfm", "-Wl,-rpath," + libdir],
                   check=True, capture_output=True)
    r = subprocess.run([str(exe), str(world)], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    out = r.stdout.splitlines()
    assert out[:len(full) + 1] == _print("full", full)
    assert out[len(full) + 1:-1] == _print("selected", sel)


def test_mapper_stage_4_matches_the_host_built_scene():
    sc = S.make_scene(20, 1500, mean_track_len=5, seed=74)
    features, pairs = _te_cpu._pairs_from_scene(sc, np.random.default_rng(3), 0.0)[:2]
    vg = S.view_graph_from_scene(sc, min_shared=10, noise_deg=0.5)
    image_ids = list(range(1, sc.C + 1))
    host_full, _ = TE.establish_full_tracks(pairs, features)
    host = TE.tracks_to_scene(TE.find_tracks_for_problem(host_full, image_ids), features, image_ids, sc.cam_intr, sc.intr_model,
                              sc.intr_params)
    assert host.P > 100
    opts = MP.GlobalMapperOptions(skip_bundle_adjustment=True)
    ok_a, a = MP.GlobalMapper(opts).Solve(vg, host)
    mapper = MP.GlobalMapper(opts)
    ok_b, b = mapper.Solve(vg, host, image_pairs=pairs, features=features)      # the scene's own tracks are not used
    assert any(line.startswith("track establishment") for line in mapper.log)
    assert ok_a and ok_b
    assert np.array_equal(a.pt_obs_begin, b.pt_obs_begin) and np.array_equal(a.obs_cam, b.obs_cam)
    assert np.array_equal(a.obs_xy, b.obs_xy)
    np.testing.assert_allclose(b.quat, a.quat, rtol=0, atol=1e-12)
    np.testing.assert_allclose(b.trans, a.trans, rtol=0, atol=1e-9)
    # skipping stage 4 uses the scene's own tracks, as before
    ok_c, c = MP.GlobalMapper(MP.GlobalMapperOptions(skip_bundle_adjustment=True, skip_track_establishment=True)).Solve(
        vg, host, image_pairs=pairs, features=features)
    assert ok_c and np.array_equal(c.obs_cam, a.obs_cam)
