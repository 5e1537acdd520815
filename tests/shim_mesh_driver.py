"""Runs ``oracle/_ref/shim_mesh`` (volrend_b200/csrc/shim/shim_mesh.cpp), the driver of the C++ ``volrend::Mesh`` and of
``VolumeRenderer`` with meshes: a :class:`Script` collects its commands, :meth:`Script.run` executes them in one
process and returns the meshes it saved and the frames it rendered."""
from __future__ import annotations

import os
import subprocess

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EXE = os.path.join(ROOT, "oracle", "_ref", "shim_mesh")


def available() -> bool:
    return os.path.exists(EXE)


def num(x) -> str:
    """``x`` as float32, written so that strtof reads back exactly that float."""
    return repr(float(np.float32(x)))


class Script:
    def __init__(self, tmp_path):
        self.dir = str(tmp_path)
        self.lines = []
        self._n = 0
        self.saves = []             # mesh directories, in save order
        self.frames = []            # (rgba path, c2w path)

    def _path(self, ext: str) -> str:
        self._n += 1
        return os.path.join(self.dir, f"shim_mesh_{self._n}{ext}")

    def add(self, *tokens) -> None:
        self.lines.append(" ".join(num(t) if isinstance(t, (float, np.floating)) else str(t) for t in tokens))

    def f32(self, arr) -> str:
        p = self._path(".f32")
        np.ascontiguousarray(arr, np.float32).tofile(p)
        return p

    def u32(self, arr) -> str:
        p = self._path(".u32")
        np.ascontiguousarray(arr, np.uint32).tofile(p)
        return p

    def file(self, data: bytes, ext: str = ".bin") -> str:
        p = self._path(ext)
        with open(p, "wb") as f:
            f.write(data)
        return p

    def save(self, i: int) -> int:
        """Saves mesh i; returns the index of the saved record in :meth:`run`'s result."""
        p = self._path(".mesh")
        os.makedirs(p)
        self.add("save", i, p)
        self.saves.append(p)
        return len(self.saves) - 1

    def render(self) -> int:
        """Renders; returns the index of the frame in :meth:`run`'s result."""
        rgba, c2w = self._path(".rgba"), self._path(".c2w")
        self.add("render", rgba, c2w)
        self.frames.append((rgba, c2w))
        return len(self.frames) - 1

    def run(self, timeout: float = 600):
        """(saved meshes as tests/mesh_io_cases.py records plus ``transform``, frames as (RGBA8 bytes, 4x3 c2w),
        stdout)."""
        path = self._path(".txt")
        with open(path, "w") as f:
            f.write("\n".join(self.lines) + "\n")
        r = subprocess.run([EXE, path], capture_output=True, text=True, timeout=timeout)
        assert r.returncode == 0, f"shim_mesh failed ({r.returncode}):\n{r.stdout}\n{r.stderr}"
        meshes = [load_saved(p) for p in self.saves]
        frames = [(np.fromfile(a, np.uint8), np.fromfile(c, np.float32).reshape(4, 3)) for a, c in self.frames]
        return meshes, frames, r.stdout


def load_saved(path: str) -> dict:
    def arr(name, dt):
        return np.fromfile(os.path.join(path, name), dt)
    f7, i3 = arr("f7.f32", np.float32), arr("i3.i32", np.int32)
    return dict(vert=arr("vert.f32", np.float32), faces=arr("faces.u32", np.uint32), name=arr("name.u8", np.uint8).tobytes(),
                scale=f7[0], translation=f7[1:4], rotation=f7[4:7], face_size=int(i3[0]), visible=bool(i3[1]),
                unlit=bool(i3[2]), transform=arr("transform.f32", np.float32))


def without_transform(rec: dict) -> dict:
    return {k: v for k, v in rec.items() if k != "transform"}
