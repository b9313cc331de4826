"""CPU: the float64 shading oracle (oracle/shade_oracle.py) against pytorch3d's index_add form of the vertex normals and
against closed-form Phong values on hand-built fragments; the compat shaders' defaults; the new C entries' argument
errors; and no CPU path through the compat renderer.  The CUDA kernels are compared with this oracle in
tests/test_gpu_shade.py."""
import ctypes
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as tF

from oracle import shade_oracle as so
from recmv_b200 import _lib


def _normals_index_add(verts, faces):
    """pytorch3d's `Meshes._compute_vertex_normals` restated in float64 torch (index_add over the three corners)."""
    v0, v1, v2 = (verts[:, faces[:, k]] for k in range(3))
    n = torch.zeros_like(verts)
    n.index_add_(1, faces[:, 1], torch.linalg.cross(v2 - v1, v0 - v1, dim=-1))
    n.index_add_(1, faces[:, 2], torch.linalg.cross(v0 - v2, v1 - v2, dim=-1))
    n.index_add_(1, faces[:, 0], torch.linalg.cross(v1 - v0, v2 - v0, dim=-1))
    return tF.normalize(n, eps=1e-6, dim=-1)


def test_oracle_normals_equal_the_index_add_form():
    g = np.random.default_rng(0)
    V, F, N = 300, 900, 3
    verts = g.normal(size=(N, V, 3))
    faces = g.integers(0, V - 20, size=(F, 3))              # the last 20 vertices are unreferenced
    faces[:10, 1] = faces[:10, 0]                            # degenerate faces with a repeated index
    ref = _normals_index_add(torch.tensor(verts), torch.tensor(faces)).numpy()
    got = so.vertex_normals(verts, faces)
    assert np.abs(got - ref).max() < 1e-12
    assert np.all(got[:, V - 20:] == 0)
    assert np.allclose(np.linalg.norm(got[:, :V - 20], axis=-1)[np.linalg.norm(ref[:, :V - 20], axis=-1) > 0.5], 1)


def test_oracle_normals_skip_faces_with_out_of_range_indices():
    verts = np.array([[[0, 0, 0], [1, 0, 0], [0, 1, 0], [5, 5, 5]]], dtype=np.float64)
    n = so.vertex_normals(verts, [[0, 1, 2], [0, 1, 7], [-1, 2, 3]])
    assert np.allclose(n[0, :3], [0, 0, 1]) and np.all(n[0, 3] == 0)


# one face in the plane z = 0 with unit normal +z; bary (0.25, 0.25, 0.5) puts the shaded point at the origin
TRI = np.array([[[-1.0, -1.0, 0.0], [1.0, -1.0, 0.0], [0.0, 1.0, 0.0]]])
UP = np.array([[[0.0, 0.0, 1.0]] * 3])
B = np.array([[[[0.25, 0.25, 0.5]]]])
P2F = np.zeros((1, 1, 1), dtype=np.int64)


def shade_one(light, eye, colors=None, **kw):
    return so.phong(P2F, B, TRI, UP, colors, [[0, 1, 2]], eye, light, **kw)[0, 0, 0]


def test_phong_light_straight_above():
    # L = N, R = N; an eye straight above sees the full highlight, one at 45 degrees (R . V = 2^-1/2)^64 = 2^-32
    assert np.allclose(shade_one([0, 0, 5], [0, 0, 3]), [1.0, 1.0, 1.0, 1.0], rtol=0, atol=1e-15)
    assert np.allclose(shade_one([0, 0, 5], [3, 0, 3]), [0.8 + 0.2 * 2.0 ** -32] * 3 + [1], rtol=0, atol=1e-15)


def test_phong_grazing_light():
    assert np.allclose(shade_one([5, 0, 0], [0, 0, 3]), [0.5, 0.5, 0.5, 1.0], rtol=0, atol=1e-15)


def test_phong_light_behind_the_surface_has_no_specular():
    # the eye below sees the mirror of a light below (R . V = 1), but cos(N, L) < 0 masks the specular term
    for eye in ([0, 0, 3], [0, 0, -3]):
        assert np.allclose(shade_one([0, 0, -5], eye), [0.5, 0.5, 0.5, 1.0], rtol=0, atol=1e-15)


def test_phong_mirror_direction_full_specular_and_colours():
    c = np.array([[[0.2, 0.4, 0.6]] * 3])
    got = shade_one([2, 0, 2], [-3, 0, 3], colors=c, light_ambient=[0.1, 0.2, 0.3], mat_specular=[1.0, 0.5, 0.25])
    dif = 0.3 / math.sqrt(2)
    want = (np.array([0.1, 0.2, 0.3]) + dif) * c[0, 0] + 0.2 * np.array([1.0, 0.5, 0.25])
    assert np.allclose(got[:3], want, rtol=0, atol=1e-14) and got[3] == 1


def test_phong_background_and_invalid_faces():
    p = np.array([[[-1, 0, 1, 5]]], dtype=np.int64)       # background, face 0, face 1 (bad index), past N F
    out = so.phong(p, np.tile(B, (1, 1, 4, 1)), TRI, UP, None, [[0, 1, 2], [0, 1, 3]], [0, 0, 3], [0, 0, 5],
                   background=(0.1, 0.2, 0.3))
    bg = np.array([0.1, 0.2, 0.3, 1.0])
    assert np.array_equal(out[0, 0, 0], bg) and np.array_equal(out[0, 0, 2], bg) and np.array_equal(out[0, 0, 3], bg)
    assert np.allclose(out[0, 0, 1], 1.0)


def test_silhouette_formula():
    out = so.silhouette(np.array([[[0, -1]]]), np.array([[[-2e-4, -1.0]]]), sigma=1e-4)
    assert np.allclose(out[0, 0, 0], [1, 1, 1, 1 / (1 + math.exp(-2))]) and np.array_equal(out[0, 0, 1], [1, 1, 1, 0])


def test_compat_defaults_are_pytorch3d_s():
    from recmv_b200.compat import MaskRender as mr
    from recmv_b200.raster import DEFAULT_LIGHTS, DEFAULT_MATERIALS
    lt, mt, bp = mr.PointLights(), mr.Materials(), mr.BlendParams()
    assert lt.location.tolist() == [[0, 1, 0]] and lt.ambient_color.tolist() == [[0.5] * 3]
    assert torch.allclose(lt.diffuse_color, torch.tensor([[0.3] * 3])) and torch.allclose(lt.specular_color,
                                                                                          torch.tensor([[0.2] * 3]))
    assert mt.ambient_color.tolist() == mt.diffuse_color.tolist() == mt.specular_color.tolist() == [[1.0] * 3]
    assert mt.shininess.tolist() == [64.0]
    assert bp.sigma == 1e-4 and bp.gamma == 1e-4 and tuple(bp.background_color) == (1.0, 1.0, 1.0)
    sh = mr.HardPhongShader(cameras="cams")
    assert sh.cameras == "cams" and sh.lights.location.tolist() == [[0, 1, 0]] and sh.materials.shininess.item() == 64
    assert mr.SoftSilhouetteShader().blend_params.sigma == 1e-4
    assert DEFAULT_LIGHTS["location"] == (0.0, 1.0, 0.0) and DEFAULT_MATERIALS["shininess"] == 64.0
    assert torch.equal(mr.TexturesVertex([torch.ones(4, 3)] * 2).verts_features_padded(), torch.ones(2, 4, 3))


class _Meshes:
    def __init__(self, verts, faces):
        self._v, self._f = verts, faces

    def verts_padded(self):
        return self._v

    def faces_list(self):
        return [self._f] * self._v.shape[0]


def test_compat_renderer_has_no_cpu_path():
    from recmv_b200.compat import MaskRender as mr
    cams = (torch.tensor([[100.0, 100.0]]), torch.tensor([[16.0, 16.0]]), torch.eye(3)[None], torch.tensor([[0, 0, 3.0]]))
    ren = mr.mask_renderer((32, 32), cams)
    ren.shader = mr.HardPhongShader(cameras=cams)
    meshes = _Meshes(torch.tensor(TRI, dtype=torch.float32), torch.tensor([[0, 1, 2]]))
    with pytest.raises(RuntimeError):
        ren(meshes)
    from recmv_b200.raster import shade_meshes, vertex_normals
    with pytest.raises(RuntimeError):
        vertex_normals(meshes._v, meshes._f)
    with pytest.raises(RuntimeError):
        shade_meshes(meshes._v, meshes._f, None, cams)


def test_new_c_entries_check_arguments_without_gpu():
    lib = _lib.load()
    nbytes = ctypes.c_size_t(0)
    assert lib.recmv_vertex_normals_workspace_bytes(10, 4, None) == -1
    assert lib.recmv_vertex_normals_workspace_bytes(-1, 4, ctypes.byref(nbytes)) == -3
    assert lib.recmv_vertex_normals_workspace_bytes(10, -4, ctypes.byref(nbytes)) == -3
    assert lib.recmv_vertex_normals_workspace_bytes(10, 1 << 30, ctypes.byref(nbytes)) == -4
    assert lib.recmv_vertex_normals(None, 1, -1, None, 0, None, None, None) == -3
    assert lib.recmv_vertex_normals(None, 0, 10, None, 0, None, None, None) == 0         # nothing to do
    assert lib.recmv_vertex_normals(None, 1, 10, None, 4, None, None, None) == -1
    assert lib.recmv_shade_phong(None, None, -1, 4, 4, None, None, None, 0, None, 0, None, None, None) == -3
    assert lib.recmv_shade_phong(None, None, 0, 4, 4, None, None, None, 0, None, 0, None, None, None) == 0
    assert lib.recmv_shade_phong(None, None, 1, 4, 4, None, None, None, 0, None, 0, None, None, None) == -1
    fake = ctypes.c_void_p(0x1000)
    assert lib.recmv_shade_phong(fake, fake, 1, 4, 4, fake, fake, None, 3, fake, 1, fake,
                                 ctypes.c_void_p(0x1004), None) == -2            # RGBA rows must be 16-byte aligned
