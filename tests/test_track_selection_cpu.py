"""Track selection (TrackEngine::FindTracksForProblem, glomap/controllers/track_establishment.cc:153-227) without a GPU:
the data-parallel formulation the device implements (``parallel_select``: saturating counters as ranks, the
max_num_tracks stop as a prefix cut) against the host loop ``find_tracks_for_problem`` on random track sets, and against a
literal transcription of the reference with its unsigned comparisons (``reference_select``) for the negative options the
host loop compares as signed values; the C ABI's argument checks; the C++ shim's TrackEngine over a recording test
double and its type-check against the glomap API."""
import ctypes as ct
import os
import subprocess

import numpy as np
import pytest

from glomap_b200 import _lib, track_establishment as TE

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MOCK = os.path.join(ROOT, "tests", "shim_mock")
U64 = (1 << 64) - 1


def _u(v):
    """int -> size_t / track_t, as C++ converts the int option in a mixed comparison."""
    return int(v) & U64


# ---- literal transcription of the reference (dicts, sets, the greedy loop) --------------------------------------------
def reference_select(tracks_full: dict, registered, o: TE.TrackEstablishmentOptions) -> dict:
    """tracks_full: {track_id: [(image_id, feature_id), ...]}.  Returns tracks_selected {track_id: restricted obs}."""
    track_lengths = []
    for track_id, obs in tracks_full.items():
        if len(obs) < _u(o.min_num_view_per_track):
            continue
        if len(obs) > _u(o.max_num_view_per_track):
            continue
        track_lengths.append((len(obs), track_id))
    track_lengths.sort(reverse=True)                                  # std::sort(rbegin, rend)
    tracks_per_camera = {int(i): 0 for i in registered}
    tracks = {}
    cameras_left = len(tracks_per_camera)
    for _, track_id in track_lengths:
        image_ids, track_temp = set(), []
        for image_id, feature_id in tracks_full[track_id]:
            if image_id not in tracks_per_camera:
                continue
            track_temp.append((image_id, feature_id))
            image_ids.add(image_id)
        if len(image_ids) < _u(o.min_num_view_per_track):
            continue
        added = False
        for image_id, _ in track_temp:
            if tracks_per_camera[image_id] > _u(o.min_num_tracks_per_view):
                continue
            tracks_per_camera[image_id] += 1
            if tracks_per_camera[image_id] > _u(o.min_num_tracks_per_view):
                cameras_left -= 1
            if not added:
                tracks[track_id] = track_temp
                added = True
        if cameras_left == 0:
            break
        if len(tracks) > _u(o.max_num_tracks):
            break
    return tracks


# ---- the data-parallel formulation (what b200sfm_tracks_select computes) -----------------------------------------------
def _ge(a, u):
    return a >= u if u < (1 << 63) else np.zeros(len(a), bool)


def _le(a, u):
    return a <= u if u < (1 << 63) else np.ones(len(a), bool)


def parallel_select(tracks: TE.Tracks, registered, o: TE.TrackEstablishmentOptions) -> np.ndarray:
    """keep mask [T]: eligibility per track, ranks of the registered observations per image in processing order, then the
    prefix cut.  No loop over tracks."""
    T = len(tracks)
    begin = np.asarray(tracks.begin, np.int64)
    L = np.diff(begin)
    reg = np.unique(np.asarray([int(i) for i in registered], np.int64))
    R = len(reg)
    img = np.asarray(tracks.obs_image, np.int64)
    ri = np.searchsorted(reg, img)
    ok = (ri < R) & (reg[np.minimum(ri, R - 1)] == img) if R else np.zeros(len(img), bool)
    t_of = np.repeat(np.arange(T), L)
    nreg = np.bincount(t_of[ok], minlength=T)
    distinct = np.bincount(np.unique(t_of[ok] * (R + 1) + ri[ok]) // (R + 1), minlength=T)
    mn, mx = _u(o.min_num_view_per_track), _u(o.max_num_view_per_track)
    elig = _ge(L, mn) & _le(L, mx) & _ge(distinct, mn)
    order = np.lexsort((tracks.track_ids, L))[::-1]                  # descending (L, id)
    pos = np.empty(T, np.int64)
    pos[order] = np.arange(T)
    if o.min_num_tracks_per_view < 0:
        sel = elig & (nreg > 0)
    else:
        m = ok & elig[t_of]
        key = np.sort(ri[m] * T + pos[t_of[m]])
        rank = np.arange(len(key)) - np.searchsorted(key, (key // T) * T)
        sel_pos = np.zeros(T, bool)
        sel_pos[key[rank <= o.min_num_tracks_per_view] % T] = True
        sel = sel_pos[pos]
    if o.max_num_tracks >= 0:
        sel_pos = sel[order]
        keep_pos = sel_pos & (np.cumsum(sel_pos) <= o.max_num_tracks + 1)
        sel = keep_pos[pos]
    return sel


# ---- random track sets ---------------------------------------------------------------------------------------------
QUOTAS = [-5, -1, 0, 1, 2, 5]
MIN_VIEWS = [0, 1, 2, 3]
MAX_TRACKS = [0, 1, 5, 50, 10_000_000]


def random_tracks(rng, T=None, I=None, max_len=9):
    """Unsorted observations, repeated images inside a track, ties in length, arbitrary uint32 image ids, ids unique."""
    T = int(rng.integers(0, 150)) if T is None else T
    I = int(rng.integers(1, 16)) if I is None else I
    image_ids = rng.choice(np.arange(1, 2**32 - 1, 7919, dtype=np.int64), I, replace=False)
    lens = rng.integers(0, max_len + 1, T)
    obs_image = rng.choice(image_ids, int(lens.sum())).astype(np.uint32)
    ids = rng.choice(2**40, T, replace=False).astype(np.uint64) if rng.random() < 0.5 else \
        (rng.choice(10 * T + 1, T, replace=False).astype(np.uint64) << np.uint64(32))
    tracks = TE.Tracks(ids, np.concatenate([[0], np.cumsum(lens)]).astype(np.int64), obs_image,
                       rng.integers(0, 1000, int(lens.sum())).astype(np.uint32))
    k = int(rng.integers(0, I + 1))
    registered = list(rng.choice(image_ids, k, replace=False)) + [2**32 - 1]           # an id no track uses
    registered += registered[:2]                                                      # repeats
    return tracks, [int(i) for i in registered]


def random_options(rng):
    return TE.TrackEstablishmentOptions(min_num_tracks_per_view=int(rng.choice(QUOTAS)),
                                        min_num_view_per_track=int(rng.choice(MIN_VIEWS)),
                                        max_num_view_per_track=int(rng.choice([3, 5, 100])),
                                        max_num_tracks=int(rng.choice(MAX_TRACKS)))


def as_dict(tracks: TE.Tracks) -> dict:
    return {int(tracks.track_ids[t]): list(zip(*[x.tolist() for x in tracks.observations(t)])) for t in range(len(tracks))}


def mask_of(tracks: TE.Tracks, selected_ids) -> np.ndarray:
    return np.isin(tracks.track_ids, np.asarray(sorted(int(i) for i in selected_ids), np.uint64))


@pytest.mark.parametrize("seed", range(300))
def test_parallel_formulation_equals_the_host_loop(seed):
    rng = np.random.default_rng(seed)
    tracks, registered = random_tracks(rng)
    o = random_options(rng)
    want = TE.find_tracks_for_problem(tracks, registered, o)
    got = parallel_select(tracks, registered, o)
    assert got.tolist() == mask_of(tracks, want.track_ids).tolist()
    assert got.sum() == len(want)


def test_the_random_cases_reach_every_rule():
    """The quota saturates images, the cap cuts, and some tracks are skipped for too few distinct registered images."""
    seen = set()
    for seed in range(300):
        rng = np.random.default_rng(seed)
        tracks, registered = random_tracks(rng)
        o = random_options(rng)
        n = int(parallel_select(tracks, registered, o).sum())
        loose = TE.TrackEstablishmentOptions(min_num_tracks_per_view=-1, min_num_view_per_track=o.min_num_view_per_track,
                                             max_num_view_per_track=o.max_num_view_per_track, max_num_tracks=-1)
        n_loose = int(parallel_select(tracks, registered, loose).sum())
        if n < n_loose:
            seen.add("quota" if o.max_num_tracks >= n_loose else "cap or quota")
        if o.max_num_tracks + 1 == n < n_loose and o.min_num_tracks_per_view < 0:
            seen.add("cap")
        if o.min_num_tracks_per_view >= 0 and o.max_num_tracks >= len(tracks) and n < n_loose:
            seen.add("quota only")
        if n == 0 and len(tracks):
            seen.add("empty")
    assert {"quota", "cap", "quota only", "empty"} <= seen, seen


def test_host_loop_equals_the_transcription_for_non_negative_options():
    for seed in range(60):
        rng = np.random.default_rng(1000 + seed)
        tracks, registered = random_tracks(rng)
        o = random_options(rng)
        ref = reference_select(as_dict(tracks), registered, o)
        got = TE.find_tracks_for_problem(tracks, registered, o)
        assert as_dict(got) == ref


@pytest.mark.parametrize("field,value", [("min_num_view_per_track", -1), ("min_num_view_per_track", -3),
                                         ("max_num_view_per_track", -1), ("max_num_view_per_track", -100),
                                         ("max_num_tracks", -1), ("max_num_tracks", -2)])
def test_negative_options_follow_the_unsigned_reference(field, value):
    """A negative min_num_view_per_track selects nothing, a negative max_num_view_per_track or max_num_tracks removes the
    bound -- the reference's int -> size_t conversion; the parallel form follows it."""
    for seed in range(25):
        rng = np.random.default_rng(2000 + seed)
        tracks, registered = random_tracks(rng, max_len=12)
        o = random_options(rng)
        setattr(o, field, value)
        ref = reference_select(as_dict(tracks), registered, o)
        assert parallel_select(tracks, registered, o).tolist() == mask_of(tracks, ref).tolist()
        if field == "min_num_view_per_track":
            assert ref == {}
    o = TE.TrackEstablishmentOptions(max_num_view_per_track=-1)
    tracks = TE.Tracks(np.array([1, 2], np.uint64), np.array([0, 3, 204]), np.array([1, 2, 3] * 68, np.uint32),
                       np.zeros(204, np.uint32))
    assert sorted(reference_select(as_dict(tracks), [1, 2, 3], o)) == [1, 2]       # the 201-view track is kept
    assert parallel_select(tracks, [1, 2, 3], o).tolist() == [True, True]


def test_hand_cases():
    tracks = TE.Tracks(np.array([10, 20, 30, 40], np.uint64), np.array([0, 4, 7, 10, 12]),
                       np.array([1, 2, 3, 4, 1, 2, 3, 2, 3, 4, 1, 2], np.uint32), np.arange(12, dtype=np.uint32))
    o = TE.TrackEstablishmentOptions
    assert parallel_select(tracks, [1, 2, 3, 4], o()).tolist() == [True, True, True, False]
    assert parallel_select(tracks, [1, 2, 3, 4], o(min_num_tracks_per_view=0)).tolist() == [True, False, False, False]
    assert parallel_select(tracks, [1, 2, 3, 4], o(max_num_tracks=0)).tolist() == [True, False, False, False]
    # quota 1: images 1-4 count 1 after track 10; track 30 (2, 3, 4) takes the second slot of 2, 3, 4; track 20 (1, 2, 3)
    # still increments image 1
    assert parallel_select(tracks, [1, 2, 3, 4], o(min_num_tracks_per_view=1)).tolist() == [True, True, True, False]
    assert parallel_select(tracks, [], o()).tolist() == [False] * 4


def test_restrict_to_images_and_subset_layout():
    tracks = TE.Tracks(np.array([5, 6], np.uint64), np.array([0, 3, 5]), np.array([1, 9, 2, 9, 9], np.uint32),
                       np.array([0, 1, 2, 3, 4], np.uint32))
    r = TE.restrict_to_images(tracks, [1, 2])
    assert r.begin.tolist() == [0, 2, 2] and r.obs_image.tolist() == [1, 2] and r.obs_feature.tolist() == [0, 2]
    s = TE._subset(tracks, np.array([1, 0]))
    assert s.track_ids.tolist() == [6, 5] and s.begin.tolist() == [0, 2, 5] and s.obs_feature.tolist() == [3, 4, 0, 1, 2]


# ---- C ABI ---------------------------------------------------------------------------------------------------------
def test_abi_rejects_null_arguments_without_a_device():
    lib = _lib.load()
    ids, begin, img = np.array([1], np.uint64), np.array([0, 1], np.int64), np.array([3], np.uint32)
    keep, num = np.zeros(1, np.uint8), ct.c_int64()
    p = lambda a: a.ctypes.data_as(ct.c_void_p)   # noqa: E731
    f = lib.b200sfm_tracks_select
    assert f(None, 1, p(ids), p(begin), p(img), 1, p(img), -1, 3, 100, 10, p(keep), ct.byref(num)) == 1
    assert f(None, 1, p(ids), None, p(img), 1, p(img), -1, 3, 100, 10, p(keep), ct.byref(num)) == 1
    assert f(None, -1, None, p(begin), None, 0, None, -1, 3, 100, 10, None, ct.byref(num)) == 1
    assert f(None, 0, None, p(begin), None, -1, None, -1, 3, 100, 10, None, None) == 1


def test_device_wrapper_checks_its_inputs_before_the_device():
    tracks = TE.Tracks(np.array([1], np.uint64), np.array([0, 2]), np.array([3], np.uint32), np.array([0], np.uint32))
    with pytest.raises(ValueError, match="begin"):
        TE.find_tracks_for_problem_device(tracks, [3], ctx=object())
    with pytest.raises(ValueError, match="range of int"):
        TE.find_tracks_for_problem_device(tracks, [3], TE.TrackEstablishmentOptions(max_num_tracks=2**31), ctx=object())


# ---- C++ shim ------------------------------------------------------------------------------------------------------
def _records(dump):
    calls, cur = [], None
    for line in dump.read_text().splitlines():
        if line.startswith("call "):
            cur = {}
            calls.append((line.split()[1], cur))
            continue
        name, n, *vals = line.split()
        assert len(vals) == int(n)
        cur[name] = [float(v) if name in ("thres", "xy1", "xy2") else int(v) for v in vals]
    return calls


def test_shim_track_engine_over_the_recording_double(tmp_path):
    lib, exe, dump = tmp_path / "libb200sfm.so", tmp_path / "track_driver", tmp_path / "dump.txt"
    subprocess.run(["/usr/bin/gcc", "-std=c99", "-O1", "-Wall", "-Werror", "-fPIC", "-shared", "-I" + os.path.join(ROOT, "include"),
                    "-o", str(lib), os.path.join(MOCK, "mock_track_select.c")], check=True, capture_output=True)
    subprocess.run(["g++", "-std=c++17", "-O1", "-Wall", "-Werror", "-I" + os.path.join(ROOT, "glomap_b200", "host"), "-o", str(exe),
                    os.path.join(MOCK, "track_driver.cc"), str(lib), "-Wl,-rpath," + str(tmp_path)], check=True, capture_output=True)
    r = subprocess.run([str(exe), "mock"], env=dict(os.environ, MOCK_DUMP=str(dump)), capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    (c1, est), (c2, sel) = _records(dump)
    assert (c1, c2) == ("tracks_establish", "tracks_select")
    # valid pairs in sorted pair-id order: (10, 20) with inlier rows 2, 0, then (20, 30) with row 1; (10, 30) is invalid
    g = lambda i, f: (i << 32) | f   # noqa: E731
    assert est["thres"] == [2.5]
    assert est["gid1"] == [g(10, 0), g(10, 1), g(20, 2)] and est["gid2"] == [g(20, 2), g(20, 0), g(30, 2)]
    assert est["xy1"] == [10, 0, 11, -1, 22, -2] and est["xy2"] == [22, -2, 20, 0, 32, -2]
    # selection: tracks in sorted id order 20, 40, 50; registered = images of registered frames (10, 20), sorted
    assert sel["options"] == [4, 1, -7, 9]
    assert sel["track_ids"] == [20, 40, 50] and sel["begin"] == [0, 3, 4, 7]
    assert sel["obs_image"] == [30, 10, 10, 20, 10, 30, 20] and sel["registered"] == [10, 20]
    out = r.stdout.splitlines()
    # the stale track 99 is cleared; the discarded track 3 stays without observations
    assert out[:3] == ["full 2", "track 3 3", "track 7 7 1:0 2:5"]
    # the double keeps t = 0, 2 (ids 20, 50); observations restricted to the registered images
    assert out[3:6] == ["selected 2", "track 20 20 10:30 10:30", "track 50 50 10:60 20:70"]
    assert out[-1] == "track driver ok"


def test_shim_track_engine_typechecks_against_the_glomap_api():
    r = subprocess.run(["g++", "-std=c++17", "-fsyntax-only", "-Wall", "-DB200SFM_WITH_GLOMAP",
                        "-I" + os.path.join(MOCK, "glomap_stub_tracks"), "-I" + os.path.join(ROOT, "glomap_b200", "host"),
                        os.path.join(MOCK, "track_typecheck.cc")], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
