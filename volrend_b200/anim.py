"""Keyframe animation without a window: the animator of the reference (``volrend_anim``, main_anim.cpp) headless.

The reference interpolates between keyframes (camera pose, focal length, render options, mesh transforms) and, when
its Render button is pressed, writes every frame of the fly-through as ``ani_out/000000.png, 000001.png, ...``
through a GLFW window and ``glReadPixels``.  Here :func:`animation_frames` restates its frame schedule and
interpolation (``AnimState::update``, main_anim.cpp:230-335) in float32, and :func:`render_animation` renders the
frames on the GPU: frames without meshes, probe or grid in one batched call with options per frame
(:func:`volrend_b200.render_frames_png`), the others in chunks through :meth:`VolumeRenderer.render_batch`.

    python -m volrend_b200.anim tree.npz keyframes.json -o ani_out/ [-w 800 -h 800] [--fps 30]
                                [--draw drawlist.npz] [--world_up 0,0,1] [--gpu N]

A keyframe file is a JSON list of objects whose keys are :class:`AnimKF` field names (``opt`` keys are
:class:`RenderOptions` field names, ``mesh_state`` maps a mesh name to ``rotation``, ``translation``, ``scale``,
``unlit``); keys left out take the defaults.
"""
from __future__ import annotations

import argparse
import copy
import dataclasses
import json
import math
import os
import sys
import warnings
from concurrent.futures import ThreadPoolExecutor
from dataclasses import dataclass, field

import numpy as np

from .host import Camera, RenderOptions, VolumeRenderer, render_frames_png, write_png_file

_F = np.float32


def _vec(v) -> np.ndarray:
    return np.array(v, dtype=np.float32).reshape(3)


# ---------------------------------------------------------------------------- glm in float32
def _dot(a, b):
    t = a * b                       # glm compute_dot: (x + y) + z of the products
    return _F(_F(t[0] + t[1]) + t[2])


def _length(v):
    return _F(np.sqrt(_dot(v, v)))


def _normalize(v):
    return v * _F(_F(1) / np.sqrt(_dot(v, v)))      # glm::normalize: v * inversesqrt(dot(v, v))


def _cross(a, b):
    return np.array([a[1] * b[2] - b[1] * a[2], a[2] * b[0] - b[2] * a[0], a[0] * b[1] - b[0] * a[1]], np.float32)


def _lerp(a, b, q):
    """lerp (main_anim.cpp:55-58): (1 - q) * a + q * b, for floats and vec3."""
    return (_F(1) - q) * a + q * b


def _lerp_int(a: int, b: int, q) -> int:
    """lerp<int>: the float result is converted back to int, truncating toward zero."""
    return int(_F(_F((_F(1) - q) * _F(a)) + _F(q * _F(b))))


def _local_sph(vec, ax, ay, az):
    """main_anim.cpp:37-45."""
    x, y, z = _dot(vec, ax), _dot(vec, ay), _dot(vec, az)
    return _F(np.arctan2(y, x)), _F(np.arcsin(z))


def _local_unsph(u, v, ax, ay, az):
    """main_anim.cpp:46-53."""
    x = _F(np.cos(v) * np.cos(u))
    y = _F(np.cos(v) * np.sin(u))
    z = _F(np.sin(v))
    return (x * ax + y * ay) + z * az


def sphc_interp(vec_start, vec_end, q, ax, ay, az, loops: int = 0) -> np.ndarray:
    """Spherical interpolation about ``az`` (main_anim.cpp:60-93): azimuth in the (ax, ay) plane, elevation
    towards az and length are interpolated linearly.  A zero-length end takes the other end's direction (both:
    az); azimuths further apart than pi go the short way round, and ``loops`` adds whole turns to the end."""
    vec_start, vec_end, q = _vec(vec_start), _vec(vec_end), _F(q)
    ax, ay, az = _vec(ax), _vec(ay), _vec(az)
    d_start, d_end = _length(vec_start), _length(vec_end)
    with np.errstate(divide="ignore", invalid="ignore"):
        su, eu = vec_start / d_start, vec_end / d_end
    if d_start == 0 and d_end == 0:
        su = eu = az
    elif d_start == 0:
        su = eu
    elif d_end == 0:
        eu = su
    u_start, v_start = _local_sph(su, ax, ay, az)
    u_end, v_end = _local_sph(eu, ax, ay, az)
    if abs(float(_F(u_start - u_end))) > math.pi:     # float difference, compared with M_PI in double
        if u_end > u_start:
            u_end = _F(float(u_end) - 2 * math.pi)
        else:
            u_start = _F(float(u_start) - 2 * math.pi)
    u_end = _F(float(u_end) + int(loops) * 2 * math.pi)
    u = _F(_lerp(u_start, u_end, q))
    v = _F(_lerp(v_start, v_end, q))
    d = _F(_lerp(d_start, d_end, q))
    return _local_unsph(u, v, ax, ay, az) * d


# ---------------------------------------------------------------------------- keyframes
@dataclass
class MeshState:
    """MeshState (main_anim.cpp:112-133): a mesh's model transform (rotation is axis-angle) and ``unlit``."""
    rotation: np.ndarray = field(default_factory=lambda: np.zeros(3, np.float32))
    translation: np.ndarray = field(default_factory=lambda: np.zeros(3, np.float32))
    scale: float = 1.0
    unlit: bool = False

    def set_mesh(self, mesh) -> None:
        mesh.rotation = _vec(self.rotation).copy()
        mesh.translation = _vec(self.translation).copy()
        mesh.scale = float(self.scale)
        mesh.unlit = bool(self.unlit)
        mesh.visible = True


@dataclass
class AnimKF:
    """One keyframe (AnimKF, main_anim.cpp:135-182): camera state, render options, the transforms of the visible
    meshes by name, and the segment configuration: ``t_max`` is the duration in seconds of the segment that ENDS at
    this keyframe, ``spherical_interp`` and ``loops`` (extra counter-clockwise turns about the world up direction)
    select how that segment moves the camera."""
    center: np.ndarray = field(default_factory=lambda: np.array([-3.55, 0.0, 3.55], np.float32))
    origin: np.ndarray = field(default_factory=lambda: np.zeros(3, np.float32))
    v_back: np.ndarray = field(default_factory=lambda: np.array([-0.7071068, 0.0, 0.7071068], np.float32))
    fx: float = 1111.0
    fy: float = 1111.0
    opt: RenderOptions = field(default_factory=RenderOptions)
    mesh_state: dict = field(default_factory=dict)
    t_max: float = 1.0
    spherical_interp: bool = True
    loops: int = 0

    def from_renderer(self, rend: VolumeRenderer) -> "AnimKF":
        """Record the renderer's state: ``v_back`` normalised, only visible meshes (main_anim.cpp:139-153)."""
        cam = rend.camera
        self.center, self.origin = _vec(cam.center).copy(), _vec(cam.origin).copy()
        self.v_back = _normalize(_vec(cam.v_back))
        self.fx, self.fy = float(_F(cam.fx)), float(_F(cam.fy))
        self.opt = copy.deepcopy(rend.options)
        self.mesh_state = {m.name: MeshState(_vec(m.rotation).copy(), _vec(m.translation).copy(), float(_F(m.scale)),
                                             bool(m.unlit)) for m in rend.meshes if m.visible}
        return self

    def to_renderer(self, rend: VolumeRenderer) -> None:
        """Apply this state (main_anim.cpp:154-168): meshes missing from ``mesh_state`` become invisible."""
        cam = rend.camera
        cam.center, cam.origin = _vec(self.center).copy(), _vec(self.origin).copy()
        cam.v_back = _normalize(_vec(self.v_back))
        cam.fx, cam.fy = float(_F(self.fx)), float(_F(self.fy))
        rend.options = copy.deepcopy(self.opt)
        for m in rend.meshes:
            if m.name not in self.mesh_state:
                m.visible = False
                continue
            self.mesh_state[m.name].set_mesh(m)

    def copy(self) -> "AnimKF":
        return copy.deepcopy(self)


def _interp(start: AnimKF, end: AnimKF, q, v_back_rend, az) -> AnimKF:
    """The state AnimState::update applies at q (main_anim.cpp:243-322).  ``v_back_rend`` is the renderer's v_back,
    i.e. that of the frame just rendered, which fixes the interpolation frame (ax, ay)."""
    curr = AnimKF()
    curr.origin = _lerp(_vec(start.origin), _vec(end.origin), q)
    start_rot, end_rot = _vec(start.opt.rot_dirs), _vec(end.opt.rot_dirs)
    ax = ay = None
    # :248-252.  The reference computes ax, ay only for spherical interpolation or meshes, and then also uses them for
    # rot_dirs (:301-303), uninitialised otherwise; here they are computed whenever one of the three needs them.
    if end.spherical_interp or end.mesh_state or (start_rot != end_rot).any():
        ax = _normalize(v_back_rend - _dot(v_back_rend, az) * az)
        ay = _normalize(_cross(az, ax))
    if end.spherical_interp:                             # :253-263; render mode always uses end.loops (:254)
        start_vec = _vec(start.center) - _vec(start.origin)
        end_vec = _vec(end.center) - _vec(end.origin)
        curr.center = curr.origin + sphc_interp(start_vec, end_vec, q, ax, ay, az, end.loops)
        curr.v_back = sphc_interp(start.v_back, end.v_back, q, ax, ay, az, end.loops)
    else:
        curr.center = _lerp(_vec(start.center), _vec(end.center), q)
        curr.v_back = _lerp(_vec(start.v_back), _vec(end.v_back), q)
    curr.fx = float(_lerp(_F(start.fx), _F(end.fx), q))
    curr.fy = float(_lerp(_F(start.fy), _F(end.fy), q))
    so, eo = start.opt, end.opt
    o = copy.deepcopy(eo)                                # :270, every other option is the end keyframe's
    o.background_brightness = float(_lerp(_F(so.background_brightness), _F(eo.background_brightness), q))
    o.step_size = float(_lerp(_F(so.step_size), _F(eo.step_size), q))
    o.stop_thresh = float(_lerp(_F(so.stop_thresh), _F(eo.stop_thresh), q))
    o.sigma_thresh = float(_lerp(_F(so.sigma_thresh), _F(eo.sigma_thresh), q))
    if so.enable_probe:                                  # :278-283
        o.probe = [float(_lerp(_F(so.probe[i]), _F(eo.probe[i]), q)) for i in range(3)]
    if eo.show_grid:                                     # :284-291
        start_depth = int(so.grid_max_depth) if so.show_grid else 0
        if start_depth != int(eo.grid_max_depth):
            o.grid_max_depth = _lerp_int(start_depth, int(eo.grid_max_depth), q)
    o.render_bbox = [float(_lerp(_F(so.render_bbox[i]), _F(eo.render_bbox[i]), q)) for i in range(6)]
    if (start_rot != end_rot).any():                     # :297-307
        o.rot_dirs = [float(v) for v in sphc_interp(start_rot, end_rot, q, ax, ay, az)]
    curr.opt = o
    curr.mesh_state = copy.deepcopy(end.mesh_state)      # :309-322
    for name, es in end.mesh_state.items():
        if name in start.mesh_state:
            ss, cs = start.mesh_state[name], curr.mesh_state[name]
            cs.rotation = sphc_interp(ss.rotation, es.rotation, q, ax, ay, az)
            cs.translation = _lerp(_vec(ss.translation), _vec(es.translation), q)
            cs.scale = float(_lerp(_F(ss.scale), _F(es.scale), q))
    curr.t_max, curr.spherical_interp, curr.loops = end.t_max, end.spherical_interp, end.loops
    return curr


def frame_camera(state: AnimKF, world_up=(0.0, 0.0, 1.0), width: int = 800, height: int = 800) -> Camera:
    """The camera VolumeRenderer.render() uses after ``state.to_renderer``."""
    cam = Camera(width, height, float(_F(state.fx)), float(_F(state.fy)))
    cam.v_world_up = _vec(world_up).copy()
    cam.center = _vec(state.center).copy()
    cam.origin = _vec(state.origin).copy()
    cam.v_back = _normalize(_vec(state.v_back))
    cam._update()
    return cam


def animation_frames(keyframes, fps: float = 30.0, world_up=(0.0, 0.0, 1.0), camera: Camera | None = None):
    """Yield ``(state, camera)`` for each frame the reference's Render button writes (``anim_from_start(false)``,
    then the loop of main_anim.cpp:1252-1262).  Frame 0 is keyframe 0.  After each written frame the animation time
    advances by 1/fps (float32) and the segment's state at q = min(t / t_max, 1) is applied, t_max being the
    segment's end keyframe's; when t >= t_max that q = 1 state is the next frame and the next segment restarts at
    t = 0, except after the last segment, whose q = 1 state is never written.  ``camera`` gives the image size of
    the yielded cameras (default 800x800).  Fewer than two keyframes: a warning, no frames (:203-205)."""
    kfs = list(keyframes)
    if len(kfs) < 2:
        warnings.warn("cannot animate with < 2 keyframes")
        return
    fps = _F(fps)
    if not (fps > 0 and np.isfinite(fps)):
        raise ValueError(f"fps must be positive, got {fps}")
    dt = _F(_F(1) / fps)
    az = _vec(world_up)
    w, h = (camera.width, camera.height) if camera is not None else (800, 800)
    state = kfs[0].copy()
    seg, t, t_max = 0, _F(0), _F(kfs[1].t_max)
    while True:
        yield state, frame_camera(state, az, w, h)
        v_back_rend = _normalize(_normalize(_vec(state.v_back)))   # to_renderer, then Camera::_update
        t_next = _F(t + dt)
        if t_next == t:
            raise ValueError(f"1/fps = {dt} no longer advances t = {t} in float32 (t_max {t_max})")
        t = t_next
        with np.errstate(divide="ignore", invalid="ignore"):
            q = min(_F(t / t_max), _F(1))
        state = _interp(kfs[seg], kfs[seg + 1], q, v_back_rend, az)
        if t >= t_max:
            if seg >= len(kfs) - 2:
                return
            seg += 1
            t, t_max = _F(0), _F(kfs[seg + 1].t_max)


# ---------------------------------------------------------------------------- rendering
# Frames per VolumeRenderer.render_batch call of render_animation: bounds its device output and host copies
# (4 B per pixel per frame, 82 MB at 800x800), of which two chunks are alive while the PNG writers drain one.
ANIM_CHUNK = 32


def _frame_view(state: AnimKF, rend: VolumeRenderer, meshes):
    """The camera, options and mesh list VolumeRenderer.render() would use for ``state`` (``to_renderer``), with the
    meshes as shallow copies of ``meshes`` so that frames share their device buffers."""
    rend.meshes = [copy.copy(m) for m in meshes]
    state.to_renderer(rend)
    return copy.deepcopy(rend.camera), rend.options, rend.meshes


def _frame_routes(states, names):
    """For each frame state, whether it goes through VolumeRenderer.render_batch (a visible mesh, the probe or the
    grid) rather than the plain per-view batch."""
    return [bool(names & set(s.mesh_state)) or bool(s.opt.enable_probe) or bool(s.opt.show_grid) for s in states]


def render_animation(tree, keyframes, fps: float, out_dir: str, *, width: int, height: int, meshes=(),
                     world_up=(0.0, 0.0, 1.0), n_threads: int = 8) -> list:
    """Write every frame of the animation to ``out_dir/%06d.png`` (main_anim.cpp:1255-1257); returns the paths.
    Frames with no visible mesh, no probe and no grid are rendered together, with one RenderOptions per frame, by
    :func:`render_frames_png`; the others in chunks of ``ANIM_CHUNK`` frames by :meth:`VolumeRenderer.render_batch`
    (meshes, probe cube and disc, grid), whose PNGs ``n_threads`` writers encode while the next chunk renders.
    Each PNG holds exactly what :meth:`VolumeRenderer.render` gives for that frame's state."""
    if not tree.is_cuda_loaded():
        tree.load_cuda()
    rend = VolumeRenderer()
    rend.meshes = list(meshes)
    rend.set(tree)
    rend.resize(width, height)
    rend.camera.v_world_up = _vec(world_up).copy()
    os.makedirs(out_dir, exist_ok=True)
    base = list(rend.meshes)
    names = {m.name for m in base}
    frames = list(animation_frames(keyframes, fps, world_up, Camera(width, height)))
    plain, full = [], []
    for i, ((state, cam), is_full) in enumerate(zip(frames, _frame_routes([s for s, _ in frames], names))):
        path = os.path.join(out_dir, "%06d.png" % i)
        if is_full:
            full.append((state, path))
        else:
            plain.append((cam, state.opt, path))
    if plain:
        render_frames_png(tree, [c for c, _, _ in plain], [o for _, o, _ in plain], [p for _, _, p in plain],
                          n_threads=n_threads)
    if full:
        for m in base:                       # upload once: every frame's copies share these buffers
            if m._vert_dev is None:
                m.update()
        _render_full_frames(rend, base, full, n_threads)
        rend.meshes = base
    return sorted([p for _, _, p in plain] + [p for _, p in full])


def _write_png(path: str, img) -> None:
    if not write_png_file(path, img):
        raise OSError(f"could not write {path}")


def _render_full_frames(rend: VolumeRenderer, meshes, full, n_threads: int) -> None:
    out, pending = None, []
    with ThreadPoolExecutor(max(int(n_threads), 1)) as pool:
        for c0 in range(0, len(full), ANIM_CHUNK):
            chunk = full[c0:c0 + ANIM_CHUNK]
            views = [_frame_view(state, rend, meshes) for state, _ in chunk]
            if out is None or out.shape[0] != len(chunk):
                out = None
            out = rend.render_batch([v[0] for v in views], [v[1] for v in views], [v[2] for v in views], out=out)
            host = out.cpu().numpy()         # synchronises: `out` may be rewritten by the next chunk
            for f in pending:                # at most two chunks of host frames alive
                f.result()
            pending = [pool.submit(_write_png, path, host[k]) for k, (_, path) in enumerate(chunk)]
        for f in pending:
            f.result()


# ---------------------------------------------------------------------------- keyframe files
_OPT_FIELDS = {f.name: f for f in dataclasses.fields(RenderOptions)}
_KF_FIELDS = [f.name for f in dataclasses.fields(AnimKF)]
_MESH_FIELDS = [f.name for f in dataclasses.fields(MeshState)]


def _num(v, what):
    if isinstance(v, bool) or not isinstance(v, (int, float)):
        raise ValueError(f"{what}: expected a number, got {v!r}")
    return float(v)


def _int(v, what):
    if isinstance(v, bool) or not isinstance(v, int):
        raise ValueError(f"{what}: expected an integer, got {v!r}")
    return v


def _bool(v, what):
    if not isinstance(v, bool):
        raise ValueError(f"{what}: expected true or false, got {v!r}")
    return v


def _nums(v, n, what, conv=_num):
    if not isinstance(v, list) or len(v) != n:
        raise ValueError(f"{what}: expected a list of {n}, got {v!r}")
    return [conv(x, what) for x in v]


def _keys(d, allowed, what):
    if not isinstance(d, dict):
        raise ValueError(f"{what}: expected an object, got {d!r}")
    bad = sorted(set(d) - set(allowed))
    if bad:
        raise ValueError(f"{what}: unknown key(s) {bad}; allowed: {sorted(allowed)}")


def _opt_from_json(d, what) -> RenderOptions:
    _keys(d, _OPT_FIELDS, what)
    o = RenderOptions()
    for k, v in d.items():
        cur = getattr(o, k)
        if isinstance(cur, bool):
            setattr(o, k, _bool(v, f"{what}.{k}"))
        elif isinstance(cur, int):
            setattr(o, k, _int(v, f"{what}.{k}"))
        elif isinstance(cur, float):
            setattr(o, k, _num(v, f"{what}.{k}"))
        else:
            conv = _int if k == "basis_minmax" else _num
            setattr(o, k, _nums(v, len(cur), f"{what}.{k}", conv))
    return o


def keyframe_from_json(d, what="keyframe") -> AnimKF:
    _keys(d, _KF_FIELDS, what)
    kf = AnimKF()
    for k in ("center", "origin", "v_back"):
        if k in d:
            setattr(kf, k, _vec(_nums(d[k], 3, f"{what}.{k}")))
    for k in ("fx", "fy", "t_max"):
        if k in d:
            setattr(kf, k, _num(d[k], f"{what}.{k}"))
    if "spherical_interp" in d:
        kf.spherical_interp = _bool(d["spherical_interp"], f"{what}.spherical_interp")
    if "loops" in d:
        kf.loops = _int(d["loops"], f"{what}.loops")
    if "opt" in d:
        kf.opt = _opt_from_json(d["opt"], f"{what}.opt")
    if "mesh_state" in d:
        _keys(d["mesh_state"], d["mesh_state"], f"{what}.mesh_state")
        for name, ms in d["mesh_state"].items():
            w = f"{what}.mesh_state[{name!r}]"
            _keys(ms, _MESH_FIELDS, w)
            st = MeshState()
            if "rotation" in ms:
                st.rotation = _vec(_nums(ms["rotation"], 3, w + ".rotation"))
            if "translation" in ms:
                st.translation = _vec(_nums(ms["translation"], 3, w + ".translation"))
            if "scale" in ms:
                st.scale = _num(ms["scale"], w + ".scale")
            if "unlit" in ms:
                st.unlit = _bool(ms["unlit"], w + ".unlit")
            kf.mesh_state[name] = st
    return kf


def keyframe_to_json(kf: AnimKF) -> dict:
    f = lambda v: [float(_F(x)) for x in np.asarray(v).reshape(-1)]
    opt = {}
    for k in _OPT_FIELDS:
        v = getattr(kf.opt, k)
        opt[k] = (list(int(x) for x in v) if k == "basis_minmax" else f(v)) if isinstance(v, (list, tuple, np.ndarray)) \
            else (v if isinstance(v, (bool, int)) else float(_F(v)))
    return {"center": f(kf.center), "origin": f(kf.origin), "v_back": f(kf.v_back), "fx": float(_F(kf.fx)),
            "fy": float(_F(kf.fy)), "opt": opt,
            "mesh_state": {n: {"rotation": f(s.rotation), "translation": f(s.translation), "scale": float(_F(s.scale)),
                               "unlit": bool(s.unlit)} for n, s in kf.mesh_state.items()},
            "t_max": float(_F(kf.t_max)), "spherical_interp": bool(kf.spherical_interp), "loops": int(kf.loops)}


def load_keyframes(path: str) -> list:
    with open(path) as fh:
        data = json.load(fh)
    if not isinstance(data, list):
        raise ValueError(f"{path}: expected a JSON list of keyframes")
    return [keyframe_from_json(d, f"keyframe {i}") for i, d in enumerate(data)]


def save_keyframes(path: str, keyframes) -> None:
    with open(path, "w") as fh:
        json.dump([keyframe_to_json(k) for k in keyframes], fh, indent=1)


# ---------------------------------------------------------------------------- CLI
def _vec3_arg(s: str):
    try:
        v = [float(x) for x in s.split(",")]
    except ValueError:
        raise argparse.ArgumentTypeError(f"expected x,y,z, got {s!r}")
    if len(v) != 3:
        raise argparse.ArgumentTypeError(f"expected x,y,z, got {s!r}")
    return v


def parse_args(argv=None):
    """The flags of volrend_anim (main_anim.cpp:1148-1168, src/opts.cpp:7-31) that concern writing frames."""
    p = argparse.ArgumentParser(prog="python -m volrend_b200.anim", add_help=False,
                                description="Render a keyframe animation to out_dir/%06d.png without a window.")
    p.add_argument("file", help="npz file storing octree data")
    p.add_argument("keyframes", help="keyframe JSON file (a list of AnimKF objects)")
    p.add_argument("-o", "--output", default="ani_out/", help="output folder (default ani_out/)")
    p.add_argument("-w", "--width", type=int, default=800, help="image width")
    p.add_argument("-h", "--height", type=int, default=800, help="image height")
    p.add_argument("--fps", type=float, default=30.0, help="frames per second of animation time")
    p.add_argument("--draw", default="", help="npz drawlist file")
    p.add_argument("--world_up", type=_vec3_arg, default=[0.0, 0.0, 1.0],
                   help="world up direction, e.g. 0,0,1=blender; ignored for NDC")
    p.add_argument("--gpu", type=int, default=-1, help="CUDA device id (-1: the current one)")
    p.add_argument("--threads", type=int, default=8, help="PNG encoder threads")
    p.add_argument("--help", action="help", help="print this help message")
    a = p.parse_args(argv)
    if a.width <= 0 or a.height <= 0:
        p.error("width and height must be positive")
    if not a.fps > 0:
        p.error("--fps must be positive")
    return a


def main(argv=None) -> int:
    a = parse_args(argv)
    import torch
    from .host import N3Tree
    from .mesh import Mesh
    if a.gpu >= 0:
        torch.cuda.set_device(a.gpu)
    kfs = load_keyframes(a.keyframes)
    tree = N3Tree(a.file)
    world_up = (0.0, 1.0, 0.0) if tree.use_ndc else a.world_up     # NDC initial camera, main_anim.cpp:1202-1212
    meshes = Mesh.open_drawlist(a.draw) if a.draw else []
    paths = render_animation(tree, kfs, a.fps, a.output, width=a.width, height=a.height, meshes=meshes,
                             world_up=world_up, n_threads=a.threads)
    print(f"wrote {len(paths)} frames to {a.output}")
    return 0


if __name__ == "__main__":
    sys.exit(main())
