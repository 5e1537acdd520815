"""`-m "not gpu"`: the animator's frame schedule and interpolation (volrend_b200/anim.py) against main_anim.cpp's
rules, restated here in float64; keyframe files and the CLI."""
import json
import math
import warnings

import numpy as np
import pytest

from volrend_b200 import RenderOptions
from volrend_b200.anim import (AnimKF, MeshState, animation_frames, keyframe_from_json, keyframe_to_json,
                               load_keyframes, parse_args, save_keyframes, sphc_interp)


# ---------------------------------------------------------------- float64 restatement of main_anim.cpp:37-93
def sph64(vs, ve, q, ax, ay, az, loops=0):
    vs, ve, ax, ay, az = (np.asarray(v, np.float64) for v in (vs, ve, ax, ay, az))
    ds, de = np.linalg.norm(vs), np.linalg.norm(ve)
    su = vs / ds if ds else None
    eu = ve / de if de else None
    if su is None and eu is None:
        su = eu = az
    elif su is None:
        su = eu
    elif eu is None:
        eu = su
    us, vs_ = math.atan2(su @ ay, su @ ax), math.asin(max(-1, min(1, su @ az)))
    ue, ve_ = math.atan2(eu @ ay, eu @ ax), math.asin(max(-1, min(1, eu @ az)))
    if abs(us - ue) > math.pi:
        if ue > us:
            ue -= 2 * math.pi
        else:
            us -= 2 * math.pi
    ue += loops * 2 * math.pi
    u, v, d = (1 - q) * us + q * ue, (1 - q) * vs_ + q * ve_, (1 - q) * ds + q * de
    return (math.cos(v) * math.cos(u) * ax + math.cos(v) * math.sin(u) * ay + math.sin(v) * az) * d


def frame_axes(v_back, az):
    az = np.asarray(az, np.float64)
    vb = np.asarray(v_back, np.float64) / np.linalg.norm(v_back)
    ax = vb - (vb @ az) * az
    ax /= np.linalg.norm(ax)
    ay = np.cross(az, ax)
    return ax, ay / np.linalg.norm(ay), az


def close_pos(a, b, tol=1e-5):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return np.abs(a - b).max() <= tol * max(1.0, np.abs(b).max())


def kf(center, v_back=None, t_max=1.0, **kw):
    k = AnimKF(t_max=t_max, **kw)
    k.center = np.array(center, np.float32)
    k.v_back = np.array(v_back if v_back is not None else -np.asarray(center) / np.linalg.norm(center), np.float32)
    return k


ORBIT = [kf([-3.5, 0, 3.5]), kf([0, -3.5, 3.5]), kf([3.5, 0, 3.5])]


# ---------------------------------------------------------------- frame schedule
def test_schedule_three_keyframes_fps4():
    frames = [s for s, _ in animation_frames(ORBIT, fps=4)]
    assert len(frames) == 8
    assert np.array_equal(frames[0].center, ORBIT[0].center)
    # frame 4 is the q = 1 state of the first segment: keyframe 1 up to rounding
    assert close_pos(frames[4].center, ORBIT[1].center)
    # keyframe 2 (the last segment's q = 1 state) is never written
    assert all(not close_pos(f.center, ORBIT[2].center, 1e-3) for f in frames)


def test_fewer_than_two_keyframes_warn_and_write_nothing():
    for ks in ([], ORBIT[:1]):
        with warnings.catch_warnings(record=True) as w:
            warnings.simplefilter("always")
            assert list(animation_frames(ks, fps=30)) == []
        assert any("< 2 keyframes" in str(x.message) for x in w)


def expected_count(t_maxes, fps):
    """Written frames from float32 accumulation: 1 (keyframe 0) + per segment the updates until t >= t_max, the
    last update of the last segment not written."""
    n = 1
    dt = np.float32(np.float32(1) / np.float32(fps))
    for tm in t_maxes:
        t, k = np.float32(0), 0
        while True:
            t = np.float32(t + dt)
            k += 1
            if t >= np.float32(tm):
                break
        n += k
    return n - 1


@pytest.mark.parametrize("t_max,fps", [(0.7, 30.0), (1.1, 24.0), (0.3, 7.0), (2.0 / 3.0, 3.0)])
def test_count_for_t_max_not_a_multiple(t_max, fps):
    ks = [kf([-3.5, 0, 3.5]), kf([0, -3.5, 3.5], t_max=t_max), kf([3.5, 0, 3.5], t_max=t_max)]
    assert len(list(animation_frames(ks, fps=fps))) == expected_count([t_max, t_max], fps)


# ---------------------------------------------------------------- sphc_interp
@pytest.mark.parametrize("loops", [0, 1, -1, 2])
@pytest.mark.parametrize("q", [0.0, 0.25, 0.5, 0.9, 1.0])
def test_sphc_interp_matches_float64(loops, q):
    az = np.array([0, 0, 1], np.float32)
    ax, ay, _ = frame_axes([-0.6, 0.2, 0.7], az)
    for vs, ve in [([-3.5, 0.1, 3.5], [0.2, -3.5, 3.0]),
                   ([-1.0, 0.01, 0.2], [-1.0, -0.01, 0.3]),            # across +-pi: the short way round
                   ([0.0, 0.0, 0.0], [1.0, 2.0, 0.5]),                   # zero-length start
                   ([1.0, 2.0, 0.5], [0.0, 0.0, 0.0]),                   # zero-length end
                   ([0.0, 0.0, 0.0], [0.0, 0.0, 0.0])]:
        got = sphc_interp(vs, ve, q, ax.astype(np.float32), ay.astype(np.float32), az, loops)
        want = sph64(vs, ve, q, ax, ay, az, loops)
        assert close_pos(got, want), (vs, ve, q, loops, got, want)


def test_wraparound_goes_short_way():
    az = np.array([0, 0, 1], np.float32)
    ax, ay = np.array([1, 0, 0], np.float32), np.array([0, 1, 0], np.float32)
    mid = sphc_interp([-1, 0.05, 0], [-1, -0.05, 0], 0.5, ax, ay, az)
    assert mid[0] < -0.99                                # through -x, not through +x
    full = sphc_interp([-1, 0.05, 0], [-1, -0.05, 0], 0.5, ax, ay, az, loops=1)
    assert close_pos(full, sph64([-1, 0.05, 0], [-1, -0.05, 0], 0.5, ax, ay, az, 1))


# ---------------------------------------------------------------- full frame states
def states64(keyframes, fps, world_up):
    """The frame states of animation_frames, computed in float64 from the same rules (main_anim.cpp:230-335)."""
    az = np.asarray(world_up, np.float64)
    out = [dict(center=keyframes[0].center, v_back=keyframes[0].v_back)]
    seg, t, dt = 0, np.float32(0), np.float32(np.float32(1) / np.float32(fps))
    prev_vb = keyframes[0].v_back
    while True:
        t = np.float32(t + dt)
        tm = np.float32(keyframes[seg + 1].t_max)
        q = float(min(np.float32(t / tm), np.float32(1)))
        s, e = keyframes[seg], keyframes[seg + 1]
        ax, ay, _ = frame_axes(prev_vb, az)
        origin = (1 - q) * s.origin.astype(np.float64) + q * e.origin
        d = {"origin": origin}
        if e.spherical_interp:
            d["center"] = origin + sph64(s.center - s.origin, e.center - e.origin, q, ax, ay, az, e.loops)
            d["v_back"] = sph64(s.v_back, e.v_back, q, ax, ay, az, e.loops)
        else:
            d["center"] = (1 - q) * s.center.astype(np.float64) + q * e.center
            d["v_back"] = (1 - q) * s.v_back.astype(np.float64) + q * e.v_back
        d["fx"] = (1 - q) * s.fx + q * e.fx
        d["step_size"] = (1 - q) * s.opt.step_size + q * e.opt.step_size
        d["bbox"] = [(1 - q) * a + q * b for a, b in zip(s.opt.render_bbox, e.opt.render_bbox)]
        srd, erd = np.asarray(s.opt.rot_dirs), np.asarray(e.opt.rot_dirs)
        d["rot_dirs"] = sph64(srd, erd, q, ax, ay, az) if (srd != erd).any() else erd
        d["mesh"] = {}
        for n, es in e.mesh_state.items():
            if n in s.mesh_state:
                ss = s.mesh_state[n]
                d["mesh"][n] = (sph64(ss.rotation, es.rotation, q, ax, ay, az),
                                (1 - q) * ss.translation.astype(np.float64) + q * es.translation,
                                (1 - q) * ss.scale + q * es.scale)
            else:
                d["mesh"][n] = (es.rotation, es.translation, es.scale)
        prev_vb = d["v_back"]
        if t >= tm:
            if seg >= len(keyframes) - 2:
                return out
            seg, t = seg + 1, np.float32(0)
        out.append(d)


def test_frame_states_match_float64():
    k0 = kf([-3.5, 0.2, 3.0], fx=1000.0)
    k0.opt = RenderOptions(step_size=1e-3, render_bbox=[0, 0, 0, 1, 1, 1], rot_dirs=[0.0, 0.0, 0.0])
    k0.mesh_state = {"a": MeshState(np.array([0.1, 0.2, 0.3], np.float32), np.array([1, 2, 3], np.float32), 1.0)}
    k1 = kf([0.1, -3.0, 3.3], fx=1200.0, t_max=0.5, loops=1)
    k1.origin = np.array([0.1, 0.0, -0.2], np.float32)
    k1.opt = RenderOptions(step_size=5e-4, render_bbox=[0.1, 0, 0.2, 0.9, 1, 0.8], rot_dirs=[0.3, -0.2, 0.5])
    k1.mesh_state = {"a": MeshState(np.array([0.4, -0.1, 0.9], np.float32), np.array([0, 1, 1], np.float32), 2.0),
                     "b": MeshState(np.array([0, 0, 1], np.float32), np.array([0, 0, 0], np.float32), 0.5)}
    k2 = kf([3.0, 0.5, 3.5], fx=900.0, t_max=0.4, spherical_interp=False)
    k2.opt = RenderOptions(step_size=2e-4, rot_dirs=[0.3, -0.2, 0.5])
    k2.mesh_state = {"b": MeshState(np.array([0, 1, 0], np.float32), np.array([1, 0, 0], np.float32), 1.5)}
    ks = [k0, k1, k2]
    got = [s for s, _ in animation_frames(ks, fps=10, world_up=(0, 0, 1))]
    want = states64(ks, 10, (0, 0, 1))
    assert len(got) == len(want) == 1 + 5 + 3      # 4 updates of the last segment, its last one not written
    for g, w in zip(got[1:], want[1:]):
        assert close_pos(g.center, w["center"]) and close_pos(g.origin, w["origin"])
        vb = np.asarray(w["v_back"], np.float64)
        assert close_pos(g.v_back / np.linalg.norm(g.v_back), vb / np.linalg.norm(vb))
        assert abs(g.fx - w["fx"]) <= 1e-5 * w["fx"]
        assert abs(g.opt.step_size - w["step_size"]) <= 1e-5 * w["step_size"]
        assert close_pos(g.opt.render_bbox, w["bbox"]) and close_pos(g.opt.rot_dirs, w["rot_dirs"])
        assert set(g.mesh_state) == set(w["mesh"])           # "a" disappears, "b" appears
        for n, (r, tr, sc) in w["mesh"].items():
            ms = g.mesh_state[n]
            assert close_pos(ms.rotation, r) and close_pos(ms.translation, tr) and abs(ms.scale - sc) <= 1e-5 * sc


def test_grid_depth_lerp_truncates_and_probe_lerp_condition():
    k0, k1 = kf([-3.5, 0, 3.5]), kf([0, -3.5, 3.5])
    k0.opt = RenderOptions(show_grid=False, probe=[0.0, 0.0, 0.0], enable_probe=False)
    k1.opt = RenderOptions(show_grid=True, grid_max_depth=7, probe=[1.0, 1.0, 1.0], enable_probe=True)
    fr = [s for s, _ in animation_frames([k0, k1, k1.copy()], fps=4)]
    # start depth 0 (no grid at the start), q = 0.25, 0.5, 0.75 -> 1.75, 3.5, 5.25 truncated
    assert [f.opt.grid_max_depth for f in fr[1:4]] == [1, 3, 5]
    assert all(f.opt.probe == [1.0, 1.0, 1.0] for f in fr[1:4])   # start has no probe: the end's, not lerped
    k0.opt.enable_probe = True
    fr = [s for s, _ in animation_frames([k0, k1, k1.copy()], fps=4)]
    assert fr[2].opt.probe == [0.5, 0.5, 0.5]


def test_camera_and_renderer_state():
    from volrend_b200 import VolumeRenderer
    from volrend_b200.mesh import Mesh
    rend = VolumeRenderer.__new__(VolumeRenderer)            # no device: only the state fields
    from volrend_b200 import Camera
    rend.camera, rend.options = Camera(), RenderOptions(step_size=3e-4)
    a, b = Mesh.Cube((0.0, 0.0, 0.0)), Mesh.Cube((0.0, 0.0, 0.0))
    a.name, b.name, b.visible = "a", "b", False
    rend.meshes = [a, b]
    rend.camera.v_back = np.array([0, 0, 2], np.float32)
    k = AnimKF().from_renderer(rend)
    assert list(k.mesh_state) == ["a"] and np.allclose(k.v_back, [0, 0, 1]) and k.opt.step_size == 3e-4
    k.mesh_state = {"b": MeshState(scale=2.0)}
    k.to_renderer(rend)
    assert not a.visible and b.visible and b.scale == 2.0


# ---------------------------------------------------------------- keyframe files and CLI
def test_json_round_trip(tmp_path):
    k = kf([-3.5, 0.25, 3.5], t_max=0.75, loops=2, spherical_interp=False)
    k.opt = RenderOptions(step_size=1.5e-4, render_bbox=[0.1, 0, 0, 1, 1, 0.9], basis_minmax=[1, 8], show_grid=True)
    k.mesh_state = {"m": MeshState(np.array([0.1, 0.2, 0.3], np.float32), np.array([1, 2, 3], np.float32), 0.5, True)}
    p = str(tmp_path / "k.json")
    save_keyframes(p, [k, AnimKF()])
    back = load_keyframes(p)
    assert keyframe_to_json(back[0]) == keyframe_to_json(k) and keyframe_to_json(back[1]) == keyframe_to_json(AnimKF())
    assert set(json.load(open(p))[0]) == {"center", "origin", "v_back", "fx", "fy", "opt", "mesh_state", "t_max",
                                         "spherical_interp", "loops"}


@pytest.mark.parametrize("bad,msg", [
    ({"centre": [0, 0, 0]}, "unknown key"),
    ({"center": [0, 0]}, "list of 3"),
    ({"fx": "big"}, "number"),
    ({"loops": 1.5}, "integer"),
    ({"spherical_interp": 1}, "true or false"),
    ({"opt": {"stepsize": 1e-3}}, "unknown key"),
    ({"opt": {"render_bbox": [0, 0, 0, 1, 1]}}, "list of 6"),
    ({"opt": {"grid_max_depth": 2.5}}, "integer"),
    ({"mesh_state": {"m": {"rot": [0, 0, 0]}}}, "unknown key"),
    ({"mesh_state": {"m": {"scale": [1]}}}, "number"),
])
def test_json_rejects(bad, msg):
    with pytest.raises(ValueError, match=msg):
        keyframe_from_json(bad)


def test_cli_parsing():
    a = parse_args(["t.npz", "k.json"])
    assert (a.output, a.width, a.height, a.fps, a.draw, a.world_up, a.gpu) == ("ani_out/", 800, 800, 30.0, "", [0, 0, 1], -1)
    a = parse_args(["t.npz", "k.json", "-o", "out", "-w", "64", "-h", "48", "--fps", "12", "--draw", "d.npz",
                    "--world_up", "0,1,0", "--gpu", "1"])
    assert (a.output, a.width, a.height, a.fps, a.draw, a.world_up, a.gpu) == ("out", 64, 48, 12.0, "d.npz", [0, 1, 0], 1)
    for bad in (["t.npz"], ["t.npz", "k.json", "--world_up", "0,1"], ["t.npz", "k.json", "-w", "0"],
                ["t.npz", "k.json", "--fps", "0"]):
        with pytest.raises(SystemExit):
            parse_args(bad)
