"""Seeded synthetic inputs of the shapes BASELINE.json names (SURVEY.md 8d): SMPL-like skeleton,
diffused skinning voxel, poses, pinhole rays, SDF grids for marching cubes.  Pure torch; used by
bench.py, the tests and the golden-vector generator (there is no network for datasets/checkpoints).
"""

import torch

# SMPL kinematic tree
PARENTS = [-1, 0, 0, 0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 9, 9, 12, 13, 14, 16, 17, 18, 19, 20, 21]

# SMPL-neutral-like rest joints (metres), baked constants (no SMPL pkl in this environment)
JOINTS = [
    [0.00, -0.24, 0.03], [0.06, -0.33, 0.02], [-0.06, -0.33, 0.02], [0.00, -0.13, 0.00],
    [0.10, -0.71, 0.02], [-0.10, -0.71, 0.02], [0.00, 0.01, 0.02], [0.09, -1.11, -0.02],
    [-0.09, -1.11, -0.02], [0.00, 0.07, 0.04], [0.11, -1.17, 0.10], [-0.11, -1.17, 0.10],
    [0.00, 0.28, 0.00], [0.08, 0.19, 0.01], [-0.08, 0.19, 0.01], [0.00, 0.37, 0.04],
    [0.18, 0.23, 0.00], [-0.18, 0.23, 0.00], [0.43, 0.22, -0.02], [-0.43, 0.22, -0.02],
    [0.68, 0.23, -0.02], [-0.68, 0.23, -0.02], [0.76, 0.22, -0.03], [-0.76, 0.22, -0.03]]


def generator(seed, device="cpu"):
    g = torch.Generator(device=device)
    g.manual_seed(int(seed))
    return g


def skeleton(device="cpu"):
    Js = torch.tensor(JOINTS, dtype=torch.float32, device=device)
    Js = Js + torch.tensor([0.0, 0.35, 0.0], device=device)  # centre the body in the bbox
    parents = torch.tensor(PARENTS, dtype=torch.long)
    init = torch.zeros(24, 3)
    init[16, 2], init[17, 2] = -0.6, 0.6  # A-pose-like shoulders
    return Js, parents, init


def skinning_voxel(shape=(65, 225, 129), seed=7, device="cpu", smooth=1):
    """ws [1,24,D,H,W]: softmax(4 randn) on a coarse lattice, trilinearly upsampled and box-smoothed
    (a stand-in for the diffused SMPL weights of model/Deformer.py:546-623)."""
    D, H, W = shape
    g = generator(seed, device)
    coarse = torch.randn((1, 24, max(D // 8, 2), max(H // 8, 2), max(W // 8, 2)), generator=g,
                         device=device) * 4.0
    ws = torch.nn.functional.interpolate(coarse, size=(D, H, W), mode="trilinear", align_corners=True)
    ws = torch.softmax(ws, dim=1)
    for _ in range(smooth):
        ws = torch.nn.functional.avg_pool3d(ws, 3, stride=1, padding=1, count_include_pad=False)
    return (ws / ws.sum(1, keepdim=True)).contiguous()


def body_points(num=6890, seed=5):
    """(verts [num,3], weights [num,24]) fp32 on CPU: a stand-in for the SMPL vertices and skinning weights that
    model/Deformer.py:594-623 diffuses into the voxel.  Points lie on capsules around the bones of skeleton() (radius
    per bone, bones chosen in proportion to their length); each point's weights go to the parent joints of its three
    nearest bones, falling off with the distance to them, so they are sparse like SMPL's.  Computed in float64 from a
    seeded CPU generator, then rounded: bit-reproducible."""
    g = generator(seed, "cpu")
    Js = skeleton()[0].double()
    par = torch.tensor(PARENTS[1:])
    a, b = Js[par], Js[1:]                                    # 23 bones: parent joint -> child joint
    length = (b - a).norm(dim=1)
    radius = torch.full((23,), 0.045, dtype=torch.float64)
    radius[[2, 5, 8, 11, 12, 14]] = 0.11                    # spine and neck bones: a thicker torso
    radius[[0, 1, 3, 4]] = 0.07                             # thighs
    bone = torch.multinomial((length + 0.05).float(), num, replacement=True, generator=g)
    t = torch.rand(num, generator=g, dtype=torch.float64)
    u = torch.randn((num, 3), generator=g, dtype=torch.float64)
    u = u / u.norm(dim=1, keepdim=True)
    verts = a[bone] + t[:, None] * (b - a)[bone] + radius[bone][:, None] * u
    # distance of every point to every bone segment -> weights of the parent joints of the three nearest bones
    ab = (b - a)[None]
    s = ((verts[:, None] - a[None]) * ab).sum(-1) / (ab * ab).sum(-1)
    d = (verts[:, None] - (a[None] + s.clamp(0, 1)[..., None] * ab)).norm(dim=-1) - radius[None]
    dn, bn = d.topk(3, dim=1, largest=False)
    wn = torch.exp(-(dn - dn[:, :1]) / 0.02)
    wn = wn / wn.sum(1, keepdim=True)
    ws = torch.zeros((num, 24), dtype=torch.float64)
    ws.index_put_((torch.arange(num)[:, None].expand(-1, 3), par[bn]), wn, accumulate=True)
    return verts.float().contiguous(), ws.float().contiguous()


def poses_trans(num_frames, seed=11, device="cpu"):
    g = generator(seed, device)
    poses = torch.randn((num_frames, 24, 3), generator=g, device=device) * 0.2
    trans = torch.randn((num_frames, 3), generator=g, device=device) * 0.05
    return poses, trans


def pinhole_rays(height=512, width=512, device="cpu", row0=0, rows=None):
    """Unit ray directions of a pinhole camera looking down +z (CameraMine.py:146-167 convention):
    fx = fy = 1.2 * width, principal point at the centre; cam_pos = (0, 0, -2.4).
    Returns dirs [rows*width, 3] for image rows [row0, row0+rows)."""
    rows = height if rows is None else rows
    fx = 1.2 * width
    v = torch.arange(row0, row0 + rows, device=device, dtype=torch.float32) + 0.5
    u = torch.arange(width, device=device, dtype=torch.float32) + 0.5
    vv, uu = torch.meshgrid(v, u, indexing="ij")
    d = torch.stack([(uu - width / 2) / fx, (vv - height / 2) / fx, torch.ones_like(uu)], -1)
    d = d / d.norm(dim=-1, keepdim=True)
    return d.reshape(-1, 3).contiguous()


CAM_POS = (0.0, 0.0, -2.4)
T_NEAR, T_FAR = 1.4, 3.4
BBOX_CENTER = (0.0, 0.0, 0.0)
BBOX_EXTEND = 2.2


def sphere_sdf_grid(res=257, num=8, seed=3, device="cpu"):
    """min_i(|x - c_i| - r_i) on a res^3 lattice over [-1,1]^3, spheres strictly inside [-0.9,0.9]^3
    (closed surfaces, no boundary crossings, occupancy ~1-2 % -- SURVEY 8d)."""
    if isinstance(res, int):
        res = (res, res, res)
    g = generator(seed, "cpu")
    c = (torch.rand((num, 3), generator=g) * 1.0 - 0.5).to(device)
    r = (torch.rand((num,), generator=g) * 0.2 + 0.15).to(device)
    axes = [torch.linspace(-1, 1, n, device=device) for n in res]
    out = None
    X, Y, Z = torch.meshgrid(*axes, indexing="ij")
    for i in range(num):
        d = torch.sqrt((X - c[i, 0]) ** 2 + (Y - c[i, 1]) ** 2 + (Z - c[i, 2]) ** 2) - r[i]
        out = d if out is None else torch.minimum(out, d)
    return out.contiguous()
