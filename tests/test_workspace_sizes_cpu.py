"""Workspace size queries, pinned.  A caller allocates what a size query returns and the run carves its buffers from
that allocation, so a query that returned fewer bytes than the run uses would let the run write past the end.  Every
query below needs no device; each row holds the status and the byte count the library returned for those extents
before the sizes were derived from the layout functions that carve the workspaces (workspace.cuh), so any change to a
size or to the order in which errors are reported fails here.  bytes is left untouched (SENTINEL) on an error.

The extents cover zero, one, ragged and production sizes (1080^2 rasterizer frames, a 257^3 marching-cubes grid,
SMPL-sized meshes of 6890 vertices and 13776 faces) and the limits on either side.  vertex_normals, knn and
mesh_adjacency ask CUB for part of their size, which needs a device, so only their cases without items to sort are
here."""
import ctypes

import pytest

from recmv_b200 import _lib

SENTINEL = 0xA5A5A5A5A5A5A5A5
NAMES = {"mc_scratch": "recmv_mc_scratch_bytes"}   # every other query is recmv_<name>_workspace_bytes

# (query, extents in C argument order with a list for an int64 array, status, bytes)
STATUS_CASES = [
    ('raster', (0, 0, 1, 1, 0), 0, 256),
    ('raster', (1, 1, 1, 1, 1), 0, 1280),
    ('raster', (3, 1001, 37, 53, 12345), 0, 338688),
    ('raster', (4, 13776, 1080, 1080, 3000000), 0, 17657344),
    ('raster', (1, 0, 1080, 1080, 0), 0, 92160),
    ('raster', (65536, 1, 1, 1, 1), 0, 7602688),
    ('raster', (1, 2147483647, 1, 1, 0), 0, 206158430976),
    ('raster', (2, 1073741824, 1, 1, 0), -4, SENTINEL),
    ('raster', (1, 1, 1, 1, 2147483647), 0, 8589935616),
    ('raster', (1, 1, 1, 1, 2147483648), -4, SENTINEL),
    ('raster', (1, 1, 44722, 44722, 0), -4, SENTINEL),
    ('raster', (1, 1, 44721, 44722, 0), -4, SENTINEL),
    ('raster', (0, 5, 2000000000, 2000000000, 7), 0, 512),
    ('raster', (-1, 1, 1, 1, 1), -3, SENTINEL),
    ('raster', (1, -1, 1, 1, 1), -3, SENTINEL),
    ('raster', (1, 1, 0, 1, 1), -3, SENTINEL),
    ('raster', (1, 1, 1, 0, 1), -3, SENTINEL),
    ('raster', (1, 1, 1, 1, -1), -3, SENTINEL),
    ('raster', (1, 1, -5, 1, 1), -3, SENTINEL),
    ('raster', (2, 2147483647, 1, 1, -1), -3, SENTINEL),
    ('raster', (-1, 2147483652, 1, 1, 2147483648), -3, SENTINEL),
    ('points_raster', (0, 0, 1, 1, 0), 0, 512),
    ('points_raster', (1, 1, 1, 1, 1), 0, 1792),
    ('points_raster', (3, 1001, 37, 53, 12345), 0, 182528),
    ('points_raster', (2, 100000, 1080, 1080, 8000000), 0, 40984064),
    ('points_raster', (65536, 1, 1, 1, 0), 0, 4194816),
    ('points_raster', (1, 2147483647, 1, 1, 0), 0, 94489281280),
    ('points_raster', (1, 2147483648, 1, 1, 0), -4, SENTINEL),
    ('points_raster', (1, 1, 1, 1, 2147483647), 0, 8589936128),
    ('points_raster', (1, 1, 1, 1, 2147483648), -4, SENTINEL),
    ('points_raster', (1, 1, 44722, 44722, 0), -4, SENTINEL),
    ('points_raster', (0, 5, 2000000000, 2000000000, 7), 0, 768),
    ('points_raster', (-1, 1, 1, 1, 1), -3, SENTINEL),
    ('points_raster', (1, -1, 1, 1, 1), -3, SENTINEL),
    ('points_raster', (1, 1, 0, 1, 1), -3, SENTINEL),
    ('points_raster', (1, 1, 1, 0, 1), -3, SENTINEL),
    ('points_raster', (1, 1, 1, 1, -1), -3, SENTINEL),
    ('points_raster', (1, 2147483648, 1, 1, -1), -3, SENTINEL),
    ('points_raster', (-1, 1, 1, 1, 2147483648), -3, SENTINEL),
    ('points_raster', (1, 2147483648, 1, 1, 2147483648), -4, SENTINEL),
    ('zbuf_probe', (0, 0, 1, 1), 0, 512),
    ('zbuf_probe', (1, 1, 1, 1), 0, 1792),
    ('zbuf_probe', (3, 1001, 37, 53), 0, 193536),
    ('zbuf_probe', (2, 20000, 1080, 1080), 0, 2744064),
    ('zbuf_probe', (1, 536870911, 8, 8), 0, 34359739392),
    ('zbuf_probe', (1, 536870912, 8, 8), -4, SENTINEL),
    ('zbuf_probe', (1, 1, 44722, 44722), -4, SENTINEL),
    ('zbuf_probe', (-1, 1, 8, 8), -3, SENTINEL),
    ('zbuf_probe', (1, -1, 8, 8), -3, SENTINEL),
    ('zbuf_probe', (1, 1, 0, 8), -3, SENTINEL),
    ('zbuf_probe', (1, 1, 8, 0), -3, SENTINEL),
    ('vertex_normals', (0, 0), 0, 0),
    ('vertex_normals', (1, 0), 0, 512),
    ('vertex_normals', (6890, 0), 0, 55296),
    ('vertex_normals', (2147483646, 0), 0, 17179869184),
    ('vertex_normals', (2147483647, 0), -4, SENTINEL),
    ('vertex_normals', (5, 715827883), -4, SENTINEL),
    ('vertex_normals', (-1, 0), -3, SENTINEL),
    ('vertex_normals', (5, -1), -3, SENTINEL),
    ('knn', (0, 0, 0), 0, 0),
    ('knn', (0, 5, 7), 0, 0),
    ('knn', (3, 0, 1000), 0, 24064),
    ('knn', (4, 0, 100000), 0, 3200000),
    ('knn', (1, 0, 2147483646), 0, 17179869184),
    ('knn', (1, 0, 2147483647), -4, SENTINEL),
    ('knn', (1, 2147483647, 1), -4, SENTINEL),
    ('knn', (2, 0, 2147483647), -4, SENTINEL),
    ('knn', (3, 0, 1431655765), -4, SENTINEL),
    ('knn', (-1, 1, 1), -3, SENTINEL),
    ('knn', (1, -1, 1), -3, SENTINEL),
    ('knn', (1, 1, -1), -3, SENTINEL),
    ('mesh_adjacency', (0, 0), 0, 0),
    ('mesh_adjacency', (1, 0), 0, 0),
    ('mesh_adjacency', (6890, 0), 0, 0),
    ('mesh_adjacency', (2147483646, 0), 0, 0),
    ('mesh_adjacency', (2147483647, 0), -4, SENTINEL),
    ('mesh_adjacency', (10, 357913942), -4, SENTINEL),
    ('mesh_adjacency', (-1, 0), -3, SENTINEL),
    ('mesh_adjacency', (1, -1), -3, SENTINEL),
    ('nricp', (0,), 0, 0),
    ('nricp', (1,), 0, 1024),
    ('nricp', (257,), 0, 19456),
    ('nricp', (6890,), 0, 496640),
    ('nricp', (2147483646,), 0, 154753040384),
    ('nricp', (2147483647,), -4, SENTINEL),
    ('nricp', (-1,), -3, SENTINEL),
    ('lap_edit', (0, 0), 0, 256),
    ('lap_edit', (1, 1), 0, 4864),
    ('lap_edit', (257, 3), 0, 41728),
    ('lap_edit', (6890, 500), 0, 997376),
    ('lap_edit', (2147483390, 0), 0, 309841588224),
    ('lap_edit', (2147483391, 0), -4, SENTINEL),
    ('lap_edit', (-1, 0), -3, SENTINEL),
    ('lap_edit', (5, -1), -3, SENTINEL),
    ('mc_scratch', (1, 1, 1), 0, 1024),
    ('mc_scratch', (31, 33, 35), 0, 148736),
    ('mc_scratch', (257, 257, 257), 0, 70153728),
    ('mc_scratch', (512, 512, 512), 0, 554697216),
    ('mc_scratch', (2000, 1000, 1000), 0, 8265625600),
    ('mc_scratch', (2000, 1000, 1001), -4, SENTINEL),
    ('mc_scratch', (0, 1, 1), -3, SENTINEL),
    ('mc_scratch', (1, 0, 1), -3, SENTINEL),
    ('mc_scratch', (1, 1, 0), -3, SENTINEL),
    ('mc_scratch', (-1, 1, 1), -3, SENTINEL),
    ('loss_points', (0, None, None), 0, 0),
    ('loss_points', (1, [0], [1]), 0, 512),
    ('loss_points', (1, [1], [1]), 0, 512),
    ('loss_points', (3, [1000, 0, 12345], [6890, 17, 255]), 0, 21760),
    ('loss_points', (9, [300, 300, 300, 300, 300, 300, 300, 300, 300], [6890, 6890, 6890, 6890, 6890, 6890, 6890, 6890, 6890]), 0, 68096),
    ('loss_points', (2, [3072, 3072], [6890, 6890]), 0, 20992),
    ('loss_points', (1, [2147483647], [0]), -3, SENTINEL),
    ('loss_points', (1, [2147483642], [5]), 0, 2248146944),
    ('loss_points', (1, [2147483642], [6]), -4, SENTINEL),
    ('loss_points', (1, [2147483648], [1]), -4, SENTINEL),
    ('loss_points', (-1, None, None), -3, SENTINEL),
    ('loss_points', (1, None, [1]), -1, SENTINEL),
    ('loss_points', (1, [1], None), -1, SENTINEL),
    ('loss_points', (2, [1, -1], [1, 1]), -3, SENTINEL),
    ('loss_points', (1, [1], [0]), -3, SENTINEL),
    ('train_rays', (0, None), 0, 0),
    ('train_rays', (1, [0]), 0, 256),
    ('train_rays', (1, [1]), 0, 1024),
    ('train_rays', (3, [1000, 0, 12345]), 0, 14336),
    ('train_rays', (9, [4096, 4096, 4096, 4096, 4096, 4096, 4096, 4096, 4096]), 0, 38656),
    ('train_rays', (2, [1166400, 1166400]), 0, 2406400),
    ('train_rays', (1, [2147483647]), 0, 2214592768),
    ('train_rays', (1, [2147483648]), -4, SENTINEL),
    ('train_rays', (-1, None), -3, SENTINEL),
    ('train_rays', (1, None), -1, SENTINEL),
    ('train_rays', (2, [5, -1]), -3, SENTINEL),
    ('surface_sample', (0, 0), 0, 0),
    ('surface_sample', (1, 1), 0, 512),
    ('surface_sample', (3, 1001), 0, 24320),
    ('surface_sample', (4, 13776), 0, 442624),
    ('surface_sample', (65535, 1), 0, 1048576),
    ('surface_sample', (65536, 1), -4, SENTINEL),
    ('surface_sample', (1, 1099511627776), 0, 8830452760576),
    ('surface_sample', (1, 1099511627777), -4, SENTINEL),
    ('surface_sample', (2, 549755813888), 0, 8830452760576),
    ('surface_sample', (2, 549755813889), -4, SENTINEL),
    ('surface_sample', (-1, 1), -3, SENTINEL),
    ('surface_sample', (1, -1), -3, SENTINEL),
    ('implicit_grad', (0, 0), 0, 512),
    ('implicit_grad', (0, 1), 0, 512),
    ('implicit_grad', (1, 1), 0, 512),
    ('implicit_grad', (6144, 2), 0, 512),
    ('implicit_grad', (16800000, 5), 0, 459776),
    ('implicit_grad', (2147483647, 1), 0, 58720768),
    ('implicit_grad', (2147483648, 1), -4, SENTINEL),
    ('implicit_grad', (-1, 1), -3, SENTINEL),
    ('implicit_grad', (1, -1), -3, SENTINEL),
    ('frame_loss', (0, 1), 0, 0),
    ('frame_loss', (1, 1), 0, 512),
    ('frame_loss', (6144, 2), 0, 512),
    ('frame_loss', (4665600, 4), 0, 218880),
    ('frame_loss', (12345, 7), 0, 1280),
    ('frame_loss', (-1, 1), -3, SENTINEL),
    ('frame_loss', (1, 0), -3, SENTINEL),
    ('frame_loss', (1, -1), -3, SENTINEL),
]
SIZE_CASES = [
    ('fragment_decode_scratch_bytes', 0, 256),
    ('fragment_decode_scratch_bytes', 1, 516),
    ('fragment_decode_scratch_bytes', 255, 516),
    ('fragment_decode_scratch_bytes', 256, 516),
    ('fragment_decode_scratch_bytes', 257, 776),
    ('fragment_decode_scratch_bytes', 1166400, 1185076),
    ('fragment_decode_scratch_bytes', 4665600, 4738756),
    ('fragment_decode_scratch_bytes', 2000000000, 2031250256),
    ('fragment_decode_scratch_bytes', -1, 256),
    ('fragment_decode_scratch_bytes', -255, 256),
    ('fragment_decode_scratch_bytes', -256, 0),
    ('fragment_decode_scratch_bytes', -257, 0),
    ('fragment_decode_scratch_bytes', -1000, 18446744073709551096),
    ('surface_solve_workspace', 0, 0),
    ('surface_solve_workspace', 1, 320),
    ('surface_solve_workspace', 3, 448),
    ('surface_solve_workspace', 3072, 196864),
    ('surface_solve_workspace', 1166400, 74649856),
    ('surface_solve_workspace', -1, 0),
    ('surface_solve_workspace', -1000, 0),
]


def _query(name, args, out):
    fn = getattr(_lib.load(), NAMES.get(name, f"recmv_{name}_workspace_bytes"))
    conv = [None if a is None else (ctypes.c_int64 * len(a))(*a) if isinstance(a, list) else a for a in args]
    return fn(*conv, out)


@pytest.mark.parametrize("name,args,status,size", STATUS_CASES)
def test_status_query(name, args, status, size):
    out = ctypes.c_size_t(SENTINEL)
    assert _query(name, args, ctypes.byref(out)) == status
    assert out.value == size


@pytest.mark.parametrize("name,args", [case[:2] for case in STATUS_CASES])
def test_null_bytes_comes_first(name, args):
    assert _query(name, args, None) == -1   # RECMV_E_NULL, whatever else is wrong with the extents


@pytest.mark.parametrize("name,n,size", SIZE_CASES)
def test_size_query(name, n, size):
    assert getattr(_lib.load(), f"recmv_{name}")(n) == size
