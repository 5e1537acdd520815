#!/usr/bin/env python
"""Generate the golden vectors under tests/golden/ from the UNMODIFIED reference CUDA renderer (oracle/_ref,
built from the reference sources by oracle/Makefile.ref).  Needs a GPU.

  python tools/make_golden.py OUT [case ...]    tests/golden/<case>.npz, the cases of tests/golden_cases.py:
      ref_f32  float RGBA of the reference's per-pixel code (tap of out[4], see oracle/ref_harness.cu)
      ref_u8   bytes written by volrend::launch_renderer (src/cuda/volrend.cu:166-172)
  python tools/make_golden.py --frames OUT       tests/golden/ref/<frame>.npz, the reference frames the GPU tests
                                                 compare with (golden_cases.REF_FRAMES)
  python tools/make_golden.py --wire OUT         tests/golden/ref/wire_*.npz, N3Tree::gen_wireframe of the trees and
                                                 cuts of tests/wire_cases.py
  python tools/make_golden.py --probe OUT        tests/golden/ref/probe_*.npz, launch_renderer with enable_probe (and
                                                 the same frame without it) for the cases of tests/probe_cases.py
  python tools/make_golden.py --mesh OUT         tests/golden/ref/mesh_*.npz, Mesh::open_drawlist_mem and
                                                 Mesh::load_mem_basic_obj of the inputs of tests/mesh_io_cases.py
                                                 (needs only oracle/_ref/libref_mesh.so, no GPU)
  python tools/make_golden.py --query OUT        tests/golden/ref/query_*.npz, the reference's query_single_from_root
                                                 (oracle/_ref/libref_query.so) on the trees and point sets of
                                                 tests/query_cases.py
  python tools/make_golden.py --edge OUT         tests/golden/ref/edge_*.npz, launch_renderer (float RGBA and bytes) of
                                                 the trees, views and options of tests/edge_cases.py

OUT receives the files; copy them to tests/golden/ (or tests/golden/ref/) and commit them.
"""
import os
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from golden_cases import (CASES, REF_FRAMES, build_case, composite_inputs, ref_frame_record,  # noqa: E402
                          ref_frame_tree, ref_frame_view)
from oracle import ref_binding as rb  # noqa: E402
from oracle import probe_oracle  # noqa: E402
from oracle import ref_wire  # noqa: E402
from probe_cases import PROBE_CASES, golden_path, probe_case  # noqa: E402
from wire_cases import WIRE_DEPTHS, golden_name, record, wire_tree  # noqa: E402
from volrend_b200 import synth  # noqa: E402


def write_case_files(name, st, ndc, tmpdir):
    os.makedirs(tmpdir, exist_ok=True)
    path = os.path.join(tmpdir, name + ".npz")
    st.save_npz(path)
    pb = path[:-4] + "_poses_bounds.npy"
    if ndc is not None:
        p = np.zeros((1, 17), np.float32)
        p[0, 0] = p[0, 6] = p[0, 12] = 1.0          # identity rotation
        p[0, 9], p[0, 4], p[0, 14] = ndc              # width, height, focal (n3tree.cpp:27-29)
        p[0, 15], p[0, 16] = 1.0, 10.0
        np.save(pb, p)
    elif os.path.exists(pb):
        os.remove(pb)
    return path


def golden_cases(out_dir, only, tmpdir):
    for name in CASES:
        if only and name not in only:
            continue
        st, W, H, pose, optkw, ndc = build_case(name)
        path = write_case_files(name, st, ndc, tmpdir)
        rt = rb.RefTree(path)
        info = rt.info()
        assert bool(info["use_ndc"]) == (ndc is not None)
        fx = synth.focal_for(W)
        c12 = synth.c2w_to_colmajor12(pose)
        opt = rb.make_options(**optkw)
        comp = composite_inputs(name, W, H)
        rin, din = comp if comp is not None else (None, None)
        f = rt.render_f32(W, H, fx, fx, c12, opt, rgba_in=rin, depth_in=din)
        u = rt.render_u8(W, H, fx, fx, c12, opt, rgba_in=rin, depth_in=din)
        rt.close()
        np.savez_compressed(os.path.join(out_dir, name + ".npz"), case=np.array(name), ref_f32=f, ref_u8=u)
        print(name, info, "alpha mean %.3f" % f[..., 3].mean(), "rgb mean %.3f" % f[..., :3].mean(), flush=True)


def reference_frames(out_dir, only, tmpdir):
    for name in REF_FRAMES:
        if only and name not in only:
            continue
        st, npz = ref_frame_tree(name)
        path = os.path.join(tmpdir, name + ".npz")
        if npz is None:
            st.save_npz(path)
        else:
            np.savez(path, **npz)
        W, H, fx, pose = ref_frame_view(name)
        c12 = synth.c2w_to_colmajor12(pose)
        rt = rb.RefTree(path)
        f = rt.render_f32(W, H, fx, fx, c12, rb.make_options())
        u = rt.render_u8(W, H, fx, fx, c12, rb.make_options())
        rt.close()
        os.remove(path)
        np.savez_compressed(os.path.join(out_dir, name + ".npz"), **ref_frame_record(name, f, u))
        print(name, f"{W}x{H}", "alpha mean %.3f" % f[..., 3].mean(), "rgb mean %.3f" % f[..., :3].mean(), flush=True)


def wireframes(out_dir, only, tmpdir):
    for name, depths in WIRE_DEPTHS.items():
        if only and name not in only:
            continue
        path = os.path.join(tmpdir, name + ".npz")
        wire_tree(name).save_npz(path)
        rt = rb.RefTree(path)
        for d in depths:
            v = ref_wire.wireframe(rt, d)
            np.savez_compressed(os.path.join(out_dir, golden_name(name, d) + ".npz"), **record(name, d, v))
            print(name, "max_depth", d, "cells", v.size // 216, flush=True)
        rt.close()
        os.remove(path)


def probe_frames(out_dir, only, tmpdir):
    for name in PROBE_CASES:
        if only and name not in only:
            continue
        st, pose, optkw, probe, disp, comp = probe_case(name)
        path = os.path.join(tmpdir, name + ".npz")
        st.save_npz(path)
        import probe_cases as pc
        fx = pc.focal()
        c12 = synth.c2w_to_colmajor12(pose)
        rin, din = comp if comp is not None else (None, None)
        u = probe_oracle.ref_render_u8(path, pc.W, pc.H, fx, fx, c12, probe_oracle.ref_options(probe, disp, **optkw),
                                       rgba_in=rin, depth_in=din)
        rt = rb.RefTree(path)
        u_off = rt.render_u8(pc.W, pc.H, fx, fx, c12, rb.make_options(**optkw), rgba_in=rin, depth_in=din)
        rt.close()
        os.remove(path)
        np.savez_compressed(os.path.join(out_dir, os.path.basename(golden_path(name))), case=np.array(name),
                            ref_u8=u, ref_u8_off=u_off)
        print(name, "disc pixels changed", int((u != u_off).any(-1).sum()), flush=True)


def mesh_loads(out_dir, only, tmpdir):
    import mesh_io_cases as mc
    from oracle import ref_mesh
    for name, (data, vis, normals) in mc.drawlist_cases().items():
        if not only or name in only:
            rec = mc.record("drawlist", data, ref_mesh.open_drawlist_mem(data, vis), vis, normals)
            np.savez_compressed(os.path.join(out_dir, "mesh_" + name + ".npz"), **rec)
            print(name, "meshes", int(rec["n"]), flush=True)
    for name, (text, normals) in mc.obj_cases().items():
        if not only or name in only:
            data = text.encode("latin-1")
            rec = mc.record("obj", data, [ref_mesh.load_mem_obj(data)], True, normals)
            np.savez_compressed(os.path.join(out_dir, "mesh_" + name + ".npz"), **rec)
            print(name, "vertices", rec["m0_vert"].size // 9, flush=True)


def queries(out_dir, only, tmpdir):
    import query_cases as qc
    from oracle import ref_query
    for name in qc.QUERY_TREES:
        if only and name not in only:
            continue
        z = qc.query_tree(name)
        path = os.path.join(tmpdir, name + ".npz")
        np.savez(path, **z)
        rt = ref_query.RefQueryTree(path)
        pts, lab = qc.all_points(name, z)
        data, cube, local, _ = rt.query(pts)
        rt.close()
        os.remove(path)
        np.savez_compressed(os.path.join(out_dir, os.path.basename(qc.golden_path(name))), case=np.array(name),
                            points=pts, set=lab, data=data.view(np.uint16), cube=cube, local=local)
        print(name, "points", len(pts), "data_dim", data.shape[1], "max cube", float(cube.max()), flush=True)


def edge_frames(out_dir, only, tmpdir):
    import edge_cases as ec
    for name in ec.TREES:
        if only and name not in only:
            continue
        st, npz = ec.edge_tree(name)
        path = os.path.join(tmpdir, name + ".npz")
        ec.write_tree_file(name, st, npz, path)
        rt = rb.RefTree(path)
        assert bool(rt.info()["use_ndc"]) == (name in ec.NDC)
        for fr in ec.frames_of(name):
            _, W, H, fx, fy, pose, kw, comp = ec.frame(fr, st)
            c12 = synth.c2w_to_colmajor12(pose)
            rin, din = comp if comp is not None else (None, None)
            f = rt.render_f32(W, H, fx, fy, c12, rb.make_options(**kw), rgba_in=rin, depth_in=din)
            u = rt.render_u8(W, H, fx, fy, c12, rb.make_options(**kw), rgba_in=rin, depth_in=din)
            np.savez_compressed(os.path.join(out_dir, os.path.basename(ec.golden_path(fr))), **ec.record(fr, f, u))
            print(fr, f"{W}x{H}", "alpha mean %.3f" % f[..., 3].mean(), "rgb mean %.3f" % f[..., :3].mean(), flush=True)
        rt.close()
        os.remove(path)


def main():
    args = sys.argv[1:]
    if "--query" in args:
        from oracle import ref_query
        args = [a for a in args if a != "--query"]
        if not args:
            raise SystemExit(__doc__)
        if not ref_query.available():
            raise SystemExit(f"{ref_query.LIB_PATH} is missing: build it with `make ref` where the reference sources are")
        os.makedirs(args[0], exist_ok=True)
        with tempfile.TemporaryDirectory() as tmpdir:
            queries(args[0], args[1:], tmpdir)
        return
    if "--mesh" in args:                # CPU only: the reference's Mesh loaders
        from oracle import ref_mesh
        args = [a for a in args if a != "--mesh"]
        if not args:
            raise SystemExit(__doc__)
        if not ref_mesh.available():
            raise SystemExit(f"{ref_mesh.LIB_PATH} is missing: build it with `make ref` where the reference sources are")
        os.makedirs(args[0], exist_ok=True)
        mesh_loads(args[0], args[1:], None)
        return
    frames = "--frames" in args
    wire = "--wire" in args
    probe = "--probe" in args
    edge = "--edge" in args
    args = [a for a in args if a not in ("--frames", "--wire", "--probe", "--edge")]
    if not args:
        raise SystemExit(__doc__)
    if not rb.available() or (wire and not ref_wire.available()) or (probe and not probe_oracle.ref_available()):
        lib_path = ref_wire.LIB_PATH if wire else probe_oracle.REF_PATH if probe else rb.LIB_PATH
        raise SystemExit(f"{lib_path} is missing: build it with `make ref` where the reference sources are")
    out_dir, only = args[0], args[1:]
    os.makedirs(out_dir, exist_ok=True)
    with tempfile.TemporaryDirectory() as tmpdir:
        run = (wireframes if wire else probe_frames if probe else reference_frames if frames else edge_frames if edge
               else golden_cases)
        run(out_dir, only, tmpdir)


if __name__ == "__main__":
    main()
