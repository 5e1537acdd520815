"""`-m "not gpu"`: the host side of batched mesh rendering: the mesh table and offsets of vr_draw_meshes_batch,
the split of a VolumeRenderer.render_batch call into runs, shallow mesh copies sharing one device buffer, the
animator's routing and chunking, and the new C-ABI calls' argument checks."""
import copy
import ctypes as C

import numpy as np
import pytest


class _FakeBuf:
    """Stands in for a CUDA tensor: the mesh table reads only numel() and data_ptr()."""

    def __init__(self, ptr, numel):
        self.ptr, self.n = ptr, numel

    def numel(self):
        return self.n

    def data_ptr(self):
        return self.ptr


def _uploaded_cube():
    from volrend_b200 import Mesh
    m = Mesh.Cube()
    m._vert_dev = _FakeBuf(0x1000, m.vert.size)
    return m


def test_mesh_table_and_offsets(built):
    from volrend_b200.mesh import _mesh_table
    a, b = _uploaded_cube(), _uploaded_cube()
    b._vert_dev = _FakeBuf(0x2000, b.vert.size)
    hidden = copy.copy(a)
    hidden.visible = False
    moved = copy.copy(a)
    moved.translation = np.array([1.0, 2.0, 3.0], np.float32)
    arr, off = _mesh_table([[a, b], [], [hidden], [moved, hidden, a]])
    assert list(off) == [0, 2, 2, 2, 4]
    assert [arr[i].vert_dev for i in range(4)] == [0x1000, 0x2000, 0x1000, 0x1000]
    assert all(arr[i].n_verts == 36 and arr[i].face_size == 3 and arr[i].faces_dev is None for i in range(4))
    model = np.array(arr[2].model[:]).reshape(4, 4)           # column-major: translation in the last column
    assert np.array_equal(model[3, :3], [1.0, 2.0, 3.0])
    assert np.array_equal(np.array(arr[3].model[:]), np.eye(4, dtype=np.float32).reshape(16))
    arr, off = _mesh_table([])
    assert list(off) == [0]


def test_shallow_copies_share_the_device_buffer(built):
    from volrend_b200.mesh import _mesh_table
    a = _uploaded_cube()
    copies = [copy.copy(a) for _ in range(5)]
    for i, c in enumerate(copies):
        c.rotation = np.array([0.0, 0.0, 0.1 * i], np.float32)
        c.unlit = i % 2 == 1
    arr, off = _mesh_table([[c] for c in copies])
    assert list(off) == list(range(6))
    assert {arr[i].vert_dev for i in range(5)} == {0x1000}
    assert [arr[i].unlit for i in range(5)] == [0, 1, 0, 1, 0]
    assert a.rotation.tolist() == [0.0, 0.0, 0.0] and not a.unlit and all(c._vert_dev is a._vert_dev for c in copies)


def test_view_runs_keep_order():
    from volrend_b200.host import _view_runs
    kinds = [True, True, False, True, False, False, False, True]
    runs = _view_runs(kinds, 2)
    assert runs == [(True, 0, 2), (False, 2, 3), (True, 3, 4), (False, 4, 6), (False, 6, 7), (True, 7, 8)]
    covered = [v for _, v0, v1 in runs for v in range(v0, v1)]
    assert covered == list(range(len(kinds)))
    assert all(all(kinds[v] == k for v in range(v0, v1)) for k, v0, v1 in runs)
    assert _view_runs([], 4) == []
    assert _view_runs([False] * 70, 32) == [(False, 0, 32), (False, 32, 64), (False, 64, 70)]


def test_anim_routing_and_frame_views(built):
    from volrend_b200 import Mesh, RenderOptions, VolumeRenderer
    from volrend_b200.anim import AnimKF, MeshState, _frame_routes, _frame_view
    states = [AnimKF(), AnimKF(), AnimKF(), AnimKF(), AnimKF()]
    states[1].mesh_state = {"Cube": MeshState(translation=np.array([0.5, 0, 0], np.float32), scale=2.0)}
    states[2].opt = RenderOptions(enable_probe=True)
    states[3].opt = RenderOptions(show_grid=True)
    states[4].mesh_state = {"NotInDrawlist": MeshState()}
    assert _frame_routes(states, {"Cube", "Sphere"}) == [False, True, True, True, False]

    rend = VolumeRenderer.__new__(VolumeRenderer)       # no device: only the state the frames take is needed
    from volrend_b200.host import Camera
    rend.camera, rend.options, rend.meshes = Camera(64, 48), RenderOptions(), []
    cube, sphere = _uploaded_cube(), Mesh.Sphere()
    sphere._vert_dev = _FakeBuf(0x3000, sphere.vert.size)
    states[1].center = np.array([1.0, 2.0, 3.0], np.float32)
    cam, opt, ms = _frame_view(states[1], rend, [cube, sphere])
    assert cam is not rend.camera and np.array_equal(cam.center, [1.0, 2.0, 3.0]) and (cam.width, cam.height) == (64, 48)
    assert opt is not states[1].opt
    assert [m.visible for m in ms] == [True, False] and ms[0].scale == 2.0 and ms[0].translation[0] == np.float32(0.5)
    assert ms[0]._vert_dev is cube._vert_dev and ms[1]._vert_dev is sphere._vert_dev
    assert cube.scale == 1.0 and cube.visible and sphere.visible      # the drawlist's meshes stay as they were


def test_anim_chunks(built, tmp_path, monkeypatch):
    """Frames with meshes go through render_batch in chunks of ANIM_CHUNK, in frame order, and reach the writers."""
    from volrend_b200 import anim
    calls, written = [], {}

    class FakeOut:
        def __init__(self, n):
            self.shape = (n, 2, 2, 4)
            self.n = n

        def cpu(self):
            return self

        def numpy(self):
            return np.arange(self.n, dtype=np.uint8).reshape(self.n, 1)

    class FakeRend:
        def render_batch(self, cams, options, meshes, out=None):
            calls.append(len(cams))
            return FakeOut(len(cams))

    monkeypatch.setattr(anim, "_frame_view", lambda state, rend, meshes: (state, None, []))
    monkeypatch.setattr(anim, "write_png_file", lambda path, img: written.__setitem__(path, int(img[0])) or True)
    full = [(i, str(tmp_path / f"{i:06d}.png")) for i in range(2 * anim.ANIM_CHUNK + 5)]
    anim._render_full_frames(FakeRend(), [], full, 3)
    assert calls == [anim.ANIM_CHUNK, anim.ANIM_CHUNK, 5]
    assert written == {p: i % anim.ANIM_CHUNK for i, p in full}


def test_batch_capi_rejects_invalid_arguments(built):
    import torch
    from volrend_b200 import _capi, lib
    l = lib()
    cams = (_capi.vr_camera * 3)()
    for c in cams:
        c.width, c.height, c.fx, c.fy = 16, 8, 10.0, 10.0
        c.c2w[0] = c.c2w[4] = c.c2w[8] = 1.0
        c.c2w[11] = 3.0
    d = _capi.vr_mesh_desc()
    d.vert_dev, d.n_verts, d.face_size = 16, 3, 3
    meshes = (_capi.vr_mesh_desc * 2)(d, d)
    dummy = C.c_void_p(16)

    def call(off, n=3, c=cams, m=meshes, img=dummy):
        o = (C.c_int32 * len(off))(*off) if off is not None else None
        return l.vr_draw_meshes_batch(c, n, m, o, img, dummy, None)

    assert call([0, 1, 1, 2], n=-1) == _capi.VR_EINVAL
    assert call(None) == _capi.VR_EINVAL and b"mesh_off" in l.vr_last_error()
    assert call([1, 1, 1, 2]) == _capi.VR_EINVAL
    assert call([0, 2, 1, 2]) == _capi.VR_EINVAL and b"decreases" in l.vr_last_error()
    assert call([0, 1, 1, 2], m=None) == _capi.VR_EINVAL
    assert call([0, 1, 1, 2], img=None) == _capi.VR_EINVAL
    assert call([0, 1, 1, 2], c=None) == _capi.VR_EINVAL
    cams[2].width = 32
    assert call([0, 1, 1, 2]) == _capi.VR_EINVAL and b"one image size" in l.vr_last_error()
    cams[2].width = 16
    cams[1].c2w[0] = 0.0                                                  # singular rotation
    assert call([0, 1, 1, 2]) == _capi.VR_EINVAL and b"singular" in l.vr_last_error()
    cams[1].c2w[0] = 1.0
    assert call([0, 0, 0, 0], n=0) == _capi.VR_OK                          # nothing to do
    o = _capi.vr_options()
    l.vr_default_options(C.byref(o))
    assert l.vr_render_composite_batch(None, cams, -1, C.byref(o), None, dummy, dummy, None, None) == _capi.VR_EINVAL
    assert l.vr_render_composite_batch_opts(None, cams, 2, o, None, None, dummy, None, None) == _capi.VR_EINVAL
    if not torch.cuda.is_available():
        assert call([0, 1, 1, 2]) == _capi.VR_ENODEVICE
        assert call([0, 0, 0, 0]) == _capi.VR_ENODEVICE                    # views without primitives, still no device
        assert b"no CPU fallback" in l.vr_last_error()
