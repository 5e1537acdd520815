"""`-m gpu`: batches with options per view (vr_render_batch_opts, vr_render_frames_png_opts) against single-view
launches, the CPU oracle and uniform batches; render_animation and its CLI against VolumeRenderer.render()."""
import os
import subprocess
import sys

import numpy as np
import pytest

from conftest import ROOT

pytestmark = pytest.mark.gpu
QUEUE, INLINE = 7, 3 + 16 * 193
TREES = ["sh1_full4", "sh4_d5", "sh9_d6", "sh16_d6", "sh25_d5", "rgba_d5", "sg9_d5", "asg4_d5"]


@pytest.fixture(scope="module")
def dev_trees(small_trees):
    from volrend_b200 import N3Tree
    return {k: (st, N3Tree.from_synth(st)) for k, st in small_trees.items()}


def _cams(W, H, n, seed=0):
    from volrend_b200 import Camera, synth
    out = []
    for p in synth.nerf_synthetic_test_poses(max(n, 8))[:n] if n <= 200 else \
            [synth.nerf_synthetic_test_poses(8)[i % 8] for i in range(n)]:
        c = Camera(W, H, synth.focal_for(W), synth.focal_for(W))
        c.set_c2w(p)
        out.append(c)
    return out


def _opts(n, basis_dim, seed=0):
    """Options that vary every field from view to view, render_depth, narrowed bbox, basis range and rot_dirs
    included."""
    from volrend_b200 import RenderOptions
    rng = np.random.default_rng(seed)
    bmax = max(basis_dim - 1, 0)
    out = []
    for i in range(n):
        lo = rng.uniform(0, 0.3, 3)
        hi = rng.uniform(0.7, 1.0, 3)
        out.append(RenderOptions(
            step_size=float(rng.choice([1e-4, 5e-4, 2e-3])), sigma_thresh=float(rng.choice([1e-2, 0.5, 5.0])),
            stop_thresh=float(rng.choice([1e-2, 0.1, 0.3])), background_brightness=float(rng.uniform(0, 1)),
            render_bbox=[float(v) for v in (lo if i % 2 else [0, 0, 0])] + [float(v) for v in (hi if i % 2 else [1, 1, 1])],
            basis_minmax=[int(i % 3 == 1), bmax - int(i % 4 == 2 and bmax > 1)],
            rot_dirs=[float(v) for v in (rng.uniform(-0.5, 0.5, 3) if i % 3 == 2 else [0, 0, 0])],
            render_depth=(i % 5 == 3)))
    return out


def _single(tree, cams, opts, tile=None, counters=False):
    import torch
    from volrend_b200 import launch_renderer
    w, h = (cams[0].width, cams[0].height) if tile is None else (tile[2], tile[3])
    u = torch.zeros((len(cams), h, w, 4), dtype=torch.uint8, device="cuda")
    f = torch.zeros((len(cams), h, w, 4), dtype=torch.float32, device="cuda")
    cnt = torch.zeros(5, dtype=torch.int64, device="cuda") if counters else None
    for i, (c, o) in enumerate(zip(cams, opts)):
        launch_renderer(tree, c, o, u[i], None, None, True, float_out=f[i], counters=cnt, tile=tile)
    torch.cuda.synchronize()
    return u.cpu().numpy(), f.cpu().numpy(), (cnt.cpu().numpy() if counters else None)


def _batch(tree, cams, opts, tile=None, counters=False):
    import torch
    from volrend_b200 import render_batch
    w, h = (cams[0].width, cams[0].height) if tile is None else (tile[2], tile[3])
    u = torch.zeros((len(cams), h, w, 4), dtype=torch.uint8, device="cuda")
    f = torch.zeros((len(cams), h, w, 4), dtype=torch.float32, device="cuda")
    cnt = torch.zeros(5, dtype=torch.int64, device="cuda") if counters else None
    render_batch(tree, cams, opts, u, float_out=f, counters=cnt, tile=tile)
    torch.cuda.synchronize()
    return u.cpu().numpy(), f.cpu().numpy(), (cnt.cpu().numpy() if counters else None)


@pytest.mark.parametrize("name", TREES)
def test_batch_opts_equals_single_view(built, dev_trees, name):
    from volrend_b200 import lib
    st, tree = dev_trees[name]
    kbd = tree.info()["kernel_basis"]
    cams = _cams(72, 56, 12)
    opts = _opts(12, max(tree.data_format.basis_dim, 1), seed=len(name))
    try:
        for variant in (INLINE, QUEUE):
            if not lib().vr_variant_supported(kbd, variant):
                continue
            lib().vr_set_variant(variant)
            for tile, counters in ((None, True), ((5, 3, 40, 37), False)):
                su, sf, sc = _single(tree, cams, opts, tile, counters)
                bu, bf, bc = _batch(tree, cams, opts, tile, counters)
                assert np.array_equal(bu, su), (name, variant, tile)
                assert np.array_equal(bf.view(np.uint32), sf.view(np.uint32)), (name, variant, tile)
                if counters:
                    assert np.array_equal(bc, sc), (name, variant, bc, sc)
    finally:
        lib().vr_set_variant(0)


def test_batch_opts_against_oracle(built, dev_trees):
    from oracle import binding as ob
    st, tree = dev_trees["sh16_d6"]
    cams, opts = _cams(48, 40, 6), _opts(6, 16, seed=3)
    _, bf, _ = _batch(tree, cams, opts)
    ot = ob.OracleTree.from_synth(st)
    for i in (0, 1, 2, 3):
        o = opts[i]
        oo = ob.make_options(step_size=o.step_size, sigma_thresh=o.sigma_thresh, stop_thresh=o.stop_thresh,
                             background_brightness=o.background_brightness, render_bbox=o.render_bbox,
                             basis_minmax=o.basis_minmax, rot_dirs=o.rot_dirs, render_depth=int(o.render_depth))
        oc = ob.make_camera(48, 40, cams[i].fx, cams[i].fy, np.ascontiguousarray(cams[i].transform).reshape(12))
        f, _, _ = ob.render(ot, oc, oo)
        assert float(np.abs(bf[i] - f).max()) <= 1e-4, i


def test_same_options_equal_uniform_batch(built, dev_trees):
    import torch
    from volrend_b200 import RenderOptions, render_batch
    _, tree = dev_trees["sh9_d6"]
    cams = _cams(64, 48, 10)
    o = RenderOptions(step_size=5e-4, background_brightness=0.3, render_bbox=[0.1, 0, 0, 1, 0.9, 1])
    u1 = torch.zeros((10, 48, 64, 4), dtype=torch.uint8, device="cuda")
    u2 = torch.ones_like(u1)
    render_batch(tree, cams, o, u1)
    render_batch(tree, cams, [o] * 10, u2)
    torch.cuda.synchronize()
    assert torch.equal(u1, u2)


def test_chunking_beyond_camera_ring(built, dev_trees):
    """More views than the camera ring holds (8192) on a tiny image: split into several launches, options advanced."""
    import torch
    from volrend_b200 import render_batch
    _, tree = dev_trees["sh4_d5"]
    n = 8192 + 300
    cams = _cams(8, 8, n)
    base = _opts(3, 4, seed=9)
    opts = [base[i % 3] for i in range(n)]
    u = torch.zeros((n, 8, 8, 4), dtype=torch.uint8, device="cuda")
    render_batch(tree, cams, opts, u)
    for k in range(3):
        ref = torch.zeros((len(range(k, n, 3)), 8, 8, 4), dtype=torch.uint8, device="cuda")
        render_batch(tree, cams[k::3], base[k], ref)
        torch.cuda.synchronize()
        assert torch.equal(u[k::3], ref), k


def test_errors(built, dev_trees):
    from volrend_b200 import _capi, lib
    _, tree = dev_trees["sh4_d5"]
    cams = _cams(16, 16, 3)
    arr = (_capi.vr_camera * 3)(*[c._as_c() for c in cams])
    assert lib().vr_render_batch_opts(tree._handle, arr, 3, None, None, None, None, None, None) == _capi.VR_EINVAL
    assert lib().vr_render_batch_opts(tree._handle, arr, -1, None, None, None, None, None, None) == _capi.VR_EINVAL
    with pytest.raises(ValueError):
        _batch(tree, cams, _opts(2, 4))


def test_frames_png_opts(built, dev_trees, tmp_path):
    from PIL import Image
    from volrend_b200 import render_frames_png
    _, tree = dev_trees["sh16_d6"]
    cams, opts = _cams(96, 64, 40), _opts(40, 16, seed=5)
    paths = [str(tmp_path / f"f{i:03d}.png") for i in range(40)]
    render_frames_png(tree, cams, opts, paths, n_threads=4)
    bu, _, _ = _batch(tree, cams, opts)
    for i in range(40):
        assert np.array_equal(np.asarray(Image.open(paths[i])), bu[i]), i


def _anim_setup(tmp_path):
    from volrend_b200 import RenderOptions
    from volrend_b200.anim import AnimKF, MeshState, save_keyframes
    kfs = []
    for i, (c, vb) in enumerate([([-3.5, 0, 3.5], None), ([0, -3.5, 3.5], None), ([3.5, 0.5, 3.0], None),
                                 ([0.5, 3.5, 3.5], None)]):
        k = AnimKF(t_max=0.25 + 0.1 * i, fx=90.0 + 5 * i, fy=90.0 + 5 * i)
        k.center = np.array(c, np.float32)
        k.v_back = (k.center / np.linalg.norm(k.center)).astype(np.float32)
        k.opt = RenderOptions(step_size=1e-4 * (1 + i), background_brightness=0.2 * i, basis_minmax=[0, 15])
        kfs.append(k)
    kfs[1].opt.enable_probe = True                     # probe in the second segment's start ...
    kfs[1].opt.probe = [0.5, 0.5, 0.5]
    kfs[2].opt.show_grid = True                        # ... the grid in its end ...
    kfs[2].opt.grid_max_depth = 3
    kfs[3].mesh_state = {"box": MeshState(np.array([0.3, 0.1, 0.2], np.float32), np.array([0.5, 0.5, 0.5], np.float32),
                                          0.3)}        # ... and a drawlist mesh in the last segment
    kfs[2].mesh_state = {"box": MeshState(np.zeros(3, np.float32), np.array([0.4, 0.5, 0.6], np.float32), 0.2)}
    kfs[2].opt.show_grid = False
    kfs[3].opt.show_grid = True
    kpath = str(tmp_path / "kf.json")
    save_keyframes(kpath, kfs)
    dl = tmp_path / "dl.npz"
    np.savez(str(dl), box="cube", box__color=np.asarray([0.1, 0.7, 0.3], np.float32))
    return kfs, kpath, str(dl)


def test_render_animation_matches_volume_renderer(built, dev_trees, tmp_path):
    from PIL import Image
    from volrend_b200 import Camera, Mesh, N3Tree, VolumeRenderer
    from volrend_b200.anim import animation_frames, render_animation
    st, _ = dev_trees["sh16_d6"]
    tree = N3Tree.from_synth(st)
    kfs, kpath, dl = _anim_setup(tmp_path)
    W, H, fps = 64, 48, 12.0
    out = str(tmp_path / "out")
    paths = render_animation(tree, kfs, fps, out, width=W, height=H, meshes=Mesh.open_drawlist(dl))
    states = list(animation_frames(kfs, fps, (0, 0, 1), Camera(W, H)))
    assert len(paths) == len(states) and paths[-1].endswith("%06d.png" % (len(states) - 1))
    rend = VolumeRenderer()
    rend.meshes = Mesh.open_drawlist(dl)
    rend.set(tree)
    rend.resize(W, H)
    kinds = set()
    for (s, _), p in zip(states, paths):
        s.to_renderer(rend)
        want = rend.render().cpu().numpy()
        assert np.array_equal(np.asarray(Image.open(p)), want), p
        kinds.add((bool(s.mesh_state), s.opt.enable_probe, s.opt.show_grid))
    assert (False, False, False) in kinds and len(kinds) >= 3
    # the CLI writes the same files
    npz = str(tmp_path / "tree.npz")
    st.save_npz(npz)
    out2 = str(tmp_path / "cli")
    env = dict(os.environ, PYTHONPATH=ROOT)
    r = subprocess.run([sys.executable, "-m", "volrend_b200.anim", npz, kpath, "-o", out2, "-w", str(W), "-h", str(H),
                        "--fps", str(fps), "--draw", dl], cwd=str(tmp_path), env=env, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    assert sorted(os.listdir(out2)) == [os.path.basename(p) for p in paths]
    for p in paths:
        assert open(p, "rb").read() == open(os.path.join(out2, os.path.basename(p)), "rb").read(), p
