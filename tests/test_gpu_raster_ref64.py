"""`-m gpu`: the CUDA mesh rasterizer (vr_draw_meshes, vr_draw_meshes_batch) against the float64 ray-cast reference
of the GL mesh pass (oracle/raster_ref64.py), on the scenes of tests/raster_ref64_cases.py.  Unambiguous pixels
must agree exactly on coverage, winner and "kept the incoming pixel", and within the reference's tolerances on depth
and colour; exact scenes must follow the fill, line and point rules with no ambiguity at all."""
import numpy as np
import pytest

from conftest import ROOT  # noqa: F401  (puts the repository root on sys.path)
import raster_ref64_cases as rc

pytestmark = pytest.mark.gpu


def _gpu_draw(s):
    import torch
    from volrend_b200 import draw_meshes
    img = torch.from_numpy(s.rgba0.copy()).cuda()
    dep = torch.from_numpy(s.depth0.copy()).cuda()
    draw_meshes(rc.camera(s), s.meshes, img, dep)
    torch.cuda.synchronize()
    return img.cpu().numpy(), dep.cpu().numpy()


@pytest.mark.parametrize("name", list(rc.SCENES))
def test_kernel_matches_reference(built, name):
    s = rc.scene(name)
    rgba, depth = _gpu_draw(s)
    ref = rc.reference(s)
    frac = rc.compare(s, ref, rgba, depth)
    print(f"{name}: ambiguous {frac:.4f} of {int((ref['covered'] | ref['ambiguous']).sum())} pixels")
    assert frac <= (s.amb_max if name in rc.ADVERSARIAL else 0.03)
    if name == "depth_zero":
        assert np.array_equal(rgba, s.rgba0) and np.array_equal(depth, s.depth0)
    elif name != "collinear":
        assert ref["covered"].sum() > 0


@pytest.mark.parametrize("name", sorted(rc.EXACT))
def test_kernel_exact_ownership(built, name):
    s = rc.EXACT[name](False)
    rgba, depth = _gpu_draw(s)
    own = rc.exact_owner(s)
    cov = depth != s.depth0
    assert np.array_equal(cov, own >= 0)
    assert np.array_equal(np.where(cov, rc.decode(rgba), -1), own)


def test_batch_with_scaled_cameras(built):
    """One vr_draw_meshes_batch launch, views with rotations scaled by 1, 1.25 and 0.8: each view matches the
    reference (the lighting moves with camPos = t / s^2)."""
    import torch
    from volrend_b200 import draw_meshes_batch
    scenes = [rc._lit_scene(False, cam_scale=k) for k in (1.0, 1.25, 0.8)]
    scenes.append(rc._specular(False))
    scenes[-1] = rc.Scene(scenes[0].W, scenes[0].H, 70.0, 70.0, scenes[-1].c2w, scenes[-1].meshes)
    imgs = torch.from_numpy(np.stack([s.rgba0 for s in scenes])).cuda()
    deps = torch.from_numpy(np.stack([s.depth0 for s in scenes])).cuda()
    draw_meshes_batch([rc.camera(s) for s in scenes], [s.meshes for s in scenes], imgs, deps)
    torch.cuda.synchronize()
    imgs, deps = imgs.cpu().numpy(), deps.cpu().numpy()
    for i, s in enumerate(scenes):
        ref = rc.reference(s)
        frac = rc.compare(s, ref, imgs[i], deps[i])
        assert frac <= 0.03 and ref["covered"].sum() > 500, (i, frac)
