"""volrend_b200 -- H100-native PlenOctree ray-marcher behind volrend's renderer surface.

The product is ``libvolrend_b200.so`` (hand-written sm_90a kernels + the C-ABI in
``include/volrend_b200.h``).  This package is the thin host-side mirror of the reference's
``N3Tree`` / ``Camera`` / ``RenderOptions`` / ``VolumeRenderer`` / ``launch_renderer`` plus
synthetic-scene generators; see DESIGN.md.
"""
from .host import (CAMERA_DEFAULT_FOCAL_LENGTH, VOLREND_GLOBAL_BASIS_MAX, Camera, DataFormat, N3Tree,
                   RenderOptions, VolumeRenderer, MultiGpuRenderer, VR_MG_TILES, VR_MG_VIEWS, image_ssim, launch_renderer, leaf_error, leaf_grads, leaf_neighbors, leaf_tv, leaf_weights, render_bands, render_bands_batch, render_batch, render_frames_host, render_frames_png, write_png_file)
from ._capi import LIB_PATH, VolrendError, lib
from .mesh import Mesh, draw_meshes, draw_meshes_batch, estimate_normals
from .compress import compress_npz
from .prune import prune_arrays, prune_npz
from .finetune import finetune, finetune_npz
from .evaluate import evaluate
from .refine import refine_npz, refine_plan
from .build import build_arrays, build_npz, grid_cells, leaf_cells
from .anim import AnimKF, animation_frames, render_animation
from .isosurface import extract_mesh, isosurface_arrays, write_obj

__all__ = ["N3Tree", "Camera", "RenderOptions", "VolumeRenderer", "DataFormat", "launch_renderer", "MultiGpuRenderer", "VR_MG_VIEWS", "VR_MG_TILES",
           "Mesh", "draw_meshes", "draw_meshes_batch", "estimate_normals", "compress_npz", "prune_arrays", "prune_npz", "leaf_weights",
           "leaf_grads", "leaf_neighbors", "leaf_tv", "image_ssim", "evaluate", "finetune", "finetune_npz", "leaf_error", "refine_plan", "refine_npz",
           "build_arrays", "build_npz", "grid_cells", "leaf_cells", "isosurface_arrays", "extract_mesh", "write_obj",
           "AnimKF", "animation_frames", "render_animation",
           "render_batch", "render_bands", "render_bands_batch", "render_frames_host", "render_frames_png", "write_png_file", "lib", "LIB_PATH", "VolrendError",
           "CAMERA_DEFAULT_FOCAL_LENGTH", "VOLREND_GLOBAL_BASIS_MAX"]
