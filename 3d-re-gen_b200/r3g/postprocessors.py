"""Mesh post-processing of stage 3 (src/2d_to_3d_models/run.py:93-95: FloaterRemover, DegenerateFaceRemover, FaceReducer
from Hunyuan3D-2/hy3dgen/shapegen/postprocessors.py:37-157) -- SURVEY.md section 8f rank 2, the step right after the
metric's end point.  The reference round-trips every mesh through pymeshlab and temporary PLY files three times; here the
marching-cubes output stays on the GPU.

  FloaterRemover         built: connected components by a lock-free union-find kernel (r3g_mesh_components), then
                         MeshLab's rule -- drop every component with fewer faces than 0.005 x the largest one -- and
                         compaction.  Components are vertex-connected (MeshLab walks face-face adjacency; the two differ
                         only at non-manifold vertices).
  DegenerateFaceRemover  the reference's is a PLY save / load round trip with no filter applied
                         (postprocessors.py:146-152): mirrored as the identity on (vertices, faces).
  FaceReducer            quadric edge-collapse decimation to 40 000 faces is MeshLab's algorithm; pymeshlab is not
                         installed here, there is neither an output nor a specification to pin against: meshes at or
                         under the limit pass through, larger ones raise NotImplementedError.  FaceReducerR3G is the
                         face reduction this project runs instead.
  FaceReducerR3G         r3g's own quadric edge-collapse decimation (r3g_mesh_decimate, include/r3g.h) with the
                         reference filter's settings fixed: boundary weight 3, normal, topology and quality guards,
                         autoclean.  Rounds of independent collapses on the GPU, deterministic; not MeshLab's collapse
                         order.
Inputs / outputs: Latent2MeshOutput (numpy or CUDA tensors) or a (vertices, faces) pair; tensors stay on their device."""
import numpy as np
import torch

from . import ops
from .vae import Latent2MeshOutput


def _unpack(mesh):
    if isinstance(mesh, Latent2MeshOutput):
        return mesh.mesh_v, mesh.mesh_f
    if hasattr(mesh, "vertices") and hasattr(mesh, "faces"):
        return mesh.vertices, mesh.faces
    return mesh


def _repack(mesh, v, f):
    if isinstance(mesh, Latent2MeshOutput):
        return Latent2MeshOutput(mesh_v=v, mesh_f=f)
    if hasattr(mesh, "vertices") and hasattr(mesh, "faces"):
        return type(mesh)(v, f)
    return v, f


def _to_tensors(v, f, device, v_dtype=None):
    """numpy arrays or tensors -> vertices (cast to v_dtype if one is given) and int32 faces as tensors on `device`."""
    if not torch.is_tensor(v):
        v, f = torch.from_numpy(np.ascontiguousarray(v)), torch.from_numpy(np.ascontiguousarray(f))
    return v.to(device=device, dtype=v_dtype), f.to(device=device, dtype=torch.int32)


def _like_input(v_in, v, f):
    """The result (v, f) as numpy arrays if the input's vertices v_in were not a tensor."""
    return (v, f) if torch.is_tensor(v_in) else (v.cpu().numpy(), f.cpu().numpy())


class FloaterRemover:
    nbfaceratio = 0.005

    def __call__(self, mesh, device="cuda"):
        v, f = _unpack(mesh)
        vt, ft = _to_tensors(v, f, device)
        if ft.shape[0] == 0:
            return mesh
        labels = ops.mesh_components(ft, vt.shape[0]).long()
        face_label = labels[ft[:, 0].long()]
        counts = torch.bincount(face_label, minlength=vt.shape[0])          # faces per component root
        keep_comp = counts >= self.nbfaceratio * counts.max()               # MeshLab: size < ratio * largest -> selected
        keep_face = keep_comp[face_label]
        keep_vert = keep_comp[labels]            # vertices of removed components (and isolated vertices: count 0) go
        new_index = torch.cumsum(keep_vert, 0, dtype=torch.int64) - 1
        v2 = vt[keep_vert]
        f2 = new_index[ft[keep_face].long()].to(torch.int32)
        return _repack(mesh, *_like_input(v, v2, f2))


class DegenerateFaceRemover:
    def __call__(self, mesh):
        return mesh


class FaceReducer:
    """MeshLab's decimation, which is not mirrored: meshes over the limit raise.  FaceReducerR3G reduces them."""

    def __call__(self, mesh, max_facenum=40000):
        _, f = _unpack(mesh)
        if max_facenum > len(f):
            return mesh
        raise NotImplementedError("quadric edge-collapse decimation (pymeshlab) is not mirrored; see the module docstring "
                                  "(FaceReducerR3G is r3g's own)")


class FaceReducerR3G:
    """Reduce a mesh to at most max_facenum faces (max_facenum - 1 or max_facenum when the collapse rules allow) on the
    GPU.  A mesh with fewer faces is returned as it is; numpy in, numpy out; tensors stay on their device."""

    def __call__(self, mesh, max_facenum=40000, device="cuda"):
        v, f = _unpack(mesh)
        if max_facenum > len(f):
            return mesh
        # `device` is where numpy input goes; tensors stay on the vertices' device
        vt, ft = _to_tensors(v, f, v.device if torch.is_tensor(v) else device, torch.float32)
        v2, f2, _ = ops.mesh_decimate(vt, ft, int(max_facenum))
        return _repack(mesh, *_like_input(v, v2, f2))
