"""GPU tests of the point rasterizer and alpha compositor (csrc/points_raster.cu, recmv_b200.raster.rasterize_points,
compat/PointRender.py) against the float64 oracle (oracle/points_oracle.py).

The oracle reads the same float32 NDC points the kernel reads, so depths compare exactly; only the squared distances
differ (float32 pixel centres).  A pixel is AMBIGUOUS when some point's d lies within MARGIN * r^2 of r^2 (its coverage
could flip; float32 d is good to about 2 r 1.2e-7, i.e. 4e-5 r^2 at r = 0.006), or its K-th and (K+1)-th depths differ by
a nonzero amount within ZTOL relative.  Ambiguous pixels are counted, printed and bounded; on all others the fragments'
idx and zbuf are bit-equal to the oracle's, dists and the images are within the bounds below, and the cotangent of the
backward is zeroed there so grad_points compares against the oracle's closed-form gradient within GRAD_TOL of its
largest entry."""
import numpy as np
import pytest
import torch
import torch.nn.functional as Fn

from oracle import points_oracle as po
from recmv_b200 import ops, raster, synth
from recmv_b200.compat.PointRender import point_renderer
from recmv_b200.model import LBSkinner

pytestmark = pytest.mark.gpu
DEV = "cuda:0"

MARGIN = 2e-4             # relative to r^2
ZTOL = 1e-6
AMBIGUOUS_SHARE = 0.02    # of the covered pixels
DISTS_TOL = 2e-4          # |d - d_ref| / r^2
IMG_TOL = 1e-3            # absolute, images in [0, max feature]
GRAD_TOL = 2e-3           # max |g - g_ref| / max |g_ref|


def compare(ndc, H, W, r, K, split=None, feats=None, label="", seed=0):
    """Forward with fragments + backward of a random cotangent, both against the oracle.  Returns (images, grad,
    counts, oracle selection)."""
    ndc = ndc.to(DEV, torch.float32).contiguous()
    N, P = ndc.shape[:2]
    G = 1 if split is None else 2
    ft = None if feats is None else torch.as_tensor(feats, dtype=torch.float32, device=DEV).reshape(N, P).contiguous()
    images, (idx, zbuf, dists), counts, ws = ops.rasterize_points(ndc, ft, H, W, r, K, split, want_fragments=True)
    n64 = ndc.double().cpu().numpy()
    f64 = None if feats is None else np.asarray(ft.cpu().double())
    ref = po.select(n64, H, W, r, K, margin=MARGIN, ztol=ZTOL)
    amb = ref["ambiguous"].reshape(-1)
    # sparse GPU fragments in (pixel, rank) order
    m = idx >= 0
    nz = m.nonzero().cpu().numpy()
    gpix = (nz[:, 0] * H + nz[:, 1]) * W + nz[:, 2]
    gi, gz, gd = idx[m].cpu().numpy(), zbuf[m].cpu().double().numpy(), dists[m].cpu().double().numpy()
    ok_g, ok_r = ~amb[gpix], ~amb[ref["pix"]]
    assert np.array_equal(gpix[ok_g], ref["pix"][ok_r]) and np.array_equal(nz[ok_g, 3], ref["rank"][ok_r])
    assert np.array_equal(gi[ok_g], ref["idx"][ok_r]) and np.array_equal(gz[ok_g], ref["z"][ok_r])
    r2 = float(r) ** 2
    ed = float(np.abs(gd[ok_g] - ref["d"][ok_r]).max() / r2) if ok_g.any() else 0.0
    assert bool((zbuf[~m] == -1).all()) and bool((dists[~m] == -1).all())
    img_ref = po.composite(ref, r, f64, split, G).reshape(G, -1)
    img = images.reshape(G, -1).cpu().double().numpy()
    ei = float(np.abs(img - img_ref)[:, ~amb].max()) if (~amb).any() else 0.0
    # backward: a random cotangent, zero on ambiguous pixels
    cot = torch.randn((G, N, H, W), generator=torch.Generator().manual_seed(seed), dtype=torch.float64)
    cot = cot * torch.as_tensor(~ref["ambiguous"])[None]
    grad = ops.rasterize_points_backward(cot.float().to(DEV), ws, counts["pairs"], N, P, H, W, r, K, split)
    gref = po.composite_grad(ref, n64, r, cot.numpy(), f64, split)
    g = grad.cpu().double().numpy()
    scale = max(float(np.abs(gref).max(initial=0.0)), 1e-30)
    eg = float(np.abs(g - gref).max(initial=0.0) / scale)
    cov = max(int((ref["count"] > 0).sum()), 1)
    print(f"[points {label}] N={N} P={P} {H}x{W} r={r} K={K} pairs={counts['pairs']} covered={counts['covered']} "
          f"skipped={counts['skipped']} ambiguous={int(amb.sum())} ({amb.sum() / cov:.2e}) dists={ed:.2e} "
          f"images={ei:.2e} grad={eg:.2e} (max |g_ref| {scale:.3e})")
    assert counts["skipped"] == ref["skipped"]
    assert counts["covered"] == int((idx[..., 0] >= 0).sum())
    assert ed < DISTS_TOL and ei < IMG_TOL and eg < GRAD_TOL, (ed, ei, eg)
    assert bool((grad[..., 2] == 0).all())
    return images, grad, counts, ref


# ---- the deformed marching-cubes sphere ----------------------------------------------------------------------------
def _skinner():
    Js, parents, init = synth.skeleton()
    ws = synth.skinning_voxel((17, 33, 21), seed=7)
    return LBSkinner(ws, [-1.1] * 3, [1.1] * 3, Js, parents, init_pose=init,
                     bbox_extend=torch.tensor(synth.BBOX_EXTEND), bbox_center=torch.tensor(synth.BBOX_CENTER)).to(DEV)


@pytest.fixture(scope="module")
def sphere_verts():
    sdf = synth.sphere_sdf_grid(257, num=8, seed=3, device=DEV)
    h = 2.0 / 256
    verts, _ = ops.mc_gpu(sdf, h, h, h, -1.0, -1.0, -1.0, 0.0)
    return verts.float().contiguous()


def deform(sk, verts, N, seed):
    poses, trans = synth.poses_trans(N, seed=seed)
    V = verts.shape[0]
    d = sk(verts.repeat(N, 1), [poses.to(DEV), trans.to(DEV)], torch.arange(N, device=DEV).repeat_interleave(V))
    return d.view(N, V, 3)


def cameras(N, H, W, seed):
    """A camera per frame in the reference's convention (R close to diag(-1, -1, 1), the body ~2.6 in front)."""
    g = np.random.default_rng(seed)
    rows = []
    for n in range(N):
        a = g.normal(size=3) * 0.15
        Kx = np.array([[0, -a[2], a[1]], [a[2], 0, -a[0]], [-a[1], a[0], 0]])
        Q = np.linalg.qr(np.eye(3) + Kx)[0]
        Q = Q * np.sign(np.diag(Q))
        R = np.diag([-1.0, -1.0, 1.0]) @ Q
        f = 0.9 * min(H, W) * (1 + 0.1 * n)
        T = np.array([0.02 * n, -0.03, 2.6 + 0.1 * n])
        rows.append(np.concatenate([[f, f * 1.02, W / 2 - 0.5 + n, H / 2 - 0.5 - n], R.reshape(-1), T]))
    return torch.tensor(np.stack(rows), dtype=torch.float32, device=DEV)


@pytest.mark.parametrize("N,H,W,seed", [(1, 1080, 1080, 1), (3, 540, 960, 2), (4, 384, 512, 3)])
def test_deformed_sphere_two_groups_against_oracle(sphere_verts, N, H, W, seed):
    with torch.no_grad():
        d = deform(_skinner(), sphere_verts, N, seed)
        ndc = raster.project_points(d, cameras(N, H, W, seed), H, W)
    P = ndc.shape[1]
    _, _, counts, ref = compare(ndc, H, W, 0.006, 50, split=P // 2, label="sphere", seed=seed)
    cov = int((ref["count"] > 0).sum())
    assert cov > 0.05 * N * H * W
    assert ref["ambiguous"].sum() < AMBIGUOUS_SHARE * cov


# ---- adversarial scenes ---------------------------------------------------------------------------------------------
def centre(col, row, H, W):
    return 1 - (2 * col + 1) / W, 1 - (2 * row + 1) / H


def test_more_than_k_points_crowd_one_pixel_with_equal_z_ties():
    g = torch.Generator().manual_seed(0)
    H, W = 16, 64
    x, y = centre(20, 5, H, W)
    P = 300
    z = torch.randint(1, 40, (P,), generator=g).double() * 0.25          # many exact depth ties
    pts = torch.stack([x + 0.01 * torch.rand(P, generator=g, dtype=torch.float64),
                       y + 0.01 * torch.rand(P, generator=g, dtype=torch.float64), z], 1)[None]
    _, _, counts, ref = compare(pts, H, W, 0.08, 50, split=120, feats=torch.rand(1, P, generator=g) + 0.5,
                                label="crowd")
    assert ref["count"].max() == 50


def test_points_behind_the_camera_at_z_zero_and_off_screen():
    H, W = 32, 32
    x, y = centre(10, 10, H, W)
    pts = torch.tensor([[[x, y, -1.0], [x, y, 0.0], [x, y, -0.0], [x + 0.05, y, 1.0], [5.0, 5.0, 1.0],
                         [float("nan"), y, 1.0], [x, y, float("nan")], [x, y, float("inf")]]])
    _, _, counts, ref = compare(pts, H, W, 0.1, 8, label="behind")
    assert counts["skipped"] == 3     # z < 0, x NaN, z NaN


def test_discs_straddling_the_image_edges_and_a_radius_over_many_tiles():
    g = torch.Generator().manual_seed(1)
    H, W = 70, 100
    P = 40
    pts = torch.stack([torch.rand(P, generator=g) * 2.4 - 1.2, torch.rand(P, generator=g) * 2.4 - 1.2,
                       torch.rand(P, generator=g) + 0.5], 1)[None]
    compare(pts, H, W, 0.05, 10, split=17, label="edges")
    compare(pts[:, :6], H, W, 0.9, 6, split=3, label="large radius")


@pytest.mark.parametrize("split", [0, 64])
def test_split_size_zero_and_all(split):
    g = torch.Generator().manual_seed(2)
    pts = torch.stack([torch.rand(64, generator=g) * 2 - 1, torch.rand(64, generator=g) * 2 - 1,
                       torch.rand(64, generator=g) + 1], 1)[None].repeat(2, 1, 1)
    images, *_ = compare(pts, 40, 48, 0.1, 12, split=split, label=f"split {split}")
    assert bool((images[1 if split == 64 else 0] == 0).all())


def test_point_on_a_pixel_centre_has_alpha_one():
    H, W = 32, 64    # centres are exact binary fractions
    x, y = centre(7, 3, H, W)
    pts = torch.tensor([[[x, y, 1.0], [x + 0.01, y, 2.0]]])
    images, grad, _, _ = compare(pts, H, W, 0.05, 4, label="centre")
    assert images[0, 0, 3, 7].item() == 1.0


def test_empty_cloud_and_one_pixel_image():
    images, grad, counts, _ = compare(torch.zeros(2, 0, 3), 8, 8, 0.1, 4, label="empty")
    assert bool((images == 0).all()) and grad.shape == (2, 0, 3) and counts["pairs"] == 0
    pts = torch.tensor([[[0.1, 0.05, 1.0], [0.3, -0.2, 0.5], [0.0, 0.0, -1.0]]])
    images, *_ = compare(pts, 1, 1, 0.5, 2, label="1x1")
    assert images.shape == (1, 1, 1, 1) and images.item() > 0


def test_pair_list_that_has_to_grow():
    g = torch.Generator().manual_seed(3)
    pts = torch.stack([torch.rand(500, generator=g) * 2 - 1, torch.rand(500, generator=g) * 2 - 1,
                       torch.rand(500, generator=g) + 1], 1)[None].to(DEV).contiguous()
    a, fa, ca, _ = ops.rasterize_points(pts, None, 64, 96, 0.08, 16, 200, want_fragments=True)
    b, fb, cb, _ = ops.rasterize_points(pts, None, 64, 96, 0.08, 16, 200, want_fragments=True, capacity=1)
    assert ca["pairs"] == cb["pairs"] > 1
    assert torch.equal(a, b) and all(torch.equal(u, v) for u, v in zip(fa, fb))


def test_bit_identical_across_runs(sphere_verts):
    H = W = 540
    with torch.no_grad():
        d = deform(_skinner(), sphere_verts, 2, 5)
        ndc = raster.project_points(d, cameras(2, H, W, 5), H, W)
    outs = []
    for _ in range(2):
        p = ndc.clone().requires_grad_()
        img = ops.RasterizePointsFunction.apply(p, None, H, W, 0.006, 50, ndc.shape[1] // 2, False)
        (img * torch.linspace(-1, 1, img.numel(), device=DEV).view_as(img)).sum().backward()
        outs.append((img.detach(), p.grad))
    assert torch.equal(outs[0][0], outs[1][0]) and torch.equal(outs[0][1], outs[1][1])
    assert outs[0][1].abs().sum() > 0


def test_argument_errors():
    pts = torch.zeros(1, 4, 3, device=DEV)
    with pytest.raises(ValueError):
        ops.rasterize_points(pts, None, 8, 8, 0.1, 65)
    with pytest.raises(RuntimeError):
        cam = cameras(1, 8, 8, 0)
        raster.rasterize_points(pts, (cam[:, :2], cam[:, 2:4], cam[:, 4:13].view(1, 3, 3), cam[:, 13:]), (8, 8), 0.1, 4,
                                features=torch.ones(1, 4, device=DEV, requires_grad=True))


# ---- a mask_loss-shaped step ------------------------------------------------------------------------------------------
def test_mask_loss_step_against_the_oracle_chain(sphere_verts):
    """Deform the template with LBSkinner, render split silhouettes through the pcRender drop-in, IoU against
    max-pooled masks (OptimGarmentNetwork.py:841-981), backward to the template vertices; the same chain with the float64
    oracle renderer (same selection) gives the same loss and template gradient."""
    N, H, W, r = 2, 360, 480, 0.006
    sk = _skinner()
    cam = cameras(N, H, W, 9)
    tmpl = sphere_verts[::3].clone().requires_grad_()
    P = tmpl.shape[0]
    split = P // 2
    ren = point_renderer((H, W), r, 50, split=True)
    ren.rasterizer.cameras = (cam[:, :2], cam[:, 2:4], cam[:, 4:13].view(N, 3, 3), cam[:, 13:16])
    d = deform(sk, tmpl, N, 9)

    class Clouds:
        def points_padded(self):
            return d

        def features_packed(self):
            return torch.ones(N * P, 1, device=DEV)

    imgs, frags = ren(Clouds(), split_size=split, all_size=P)
    assert frags is None and imgs[0].shape == (N, H, W, 1)
    rad = int(np.round(ren.rasterizer.raster_settings.radius / 2.0 * min(H, W) / 1.2))
    gts = [Fn.max_pool2d((torch.roll(im.detach()[..., 0], 3, 2) > 0.5).float()[:, None], 2 * rad + 1, 1, rad)[:, 0]
           for im in imgs]

    def iou_loss(images, masks):
        loss = 0.0
        for im, gt in zip(images, masks):
            m = im[..., -1]
            loss = loss + (1 - (m * gt).view(N, -1).sum(1) / (m + gt - m * gt).abs().view(N, -1).sum(1)).mean()
        return loss

    loss = iou_loss(imgs, gts)
    gd, = torch.autograd.grad(loss, d, retain_graph=True)
    gv, = torch.autograd.grad(d, tmpl, gd, retain_graph=True)
    # the oracle chain: float64 projection + composite of the same selection
    with torch.no_grad():
        sel = po.select(raster.project_points(d, cam, H, W).double().cpu().numpy(), H, W, r, 50)
    d64 = d.detach().double().cpu().requires_grad_()
    c64 = cam.double().cpu()
    v = torch.bmm(d64, c64[:, 4:13].view(N, 3, 3)) + c64[:, None, 13:16]
    sx = c64[:, None, 2] - c64[:, None, 0] * v[..., 0] / v[..., 2]
    sy = c64[:, None, 3] - c64[:, None, 1] * v[..., 1] / v[..., 2]
    ndc64 = torch.stack([1 - (2 * sx + 1) / W, 1 - (2 * sy + 1) / H, v[..., 2]], -1)
    ref_imgs = po.composite_torch(sel, ndc64, r, None, split, 2)
    loss64 = iou_loss([im[..., None] for im in ref_imgs], [gt.double().cpu() for gt in gts])
    gd64, = torch.autograd.grad(loss64, d64)
    gv_ref, = torch.autograd.grad(d, tmpl, gd64.float().to(DEV))
    el = abs(loss.item() - loss64.item())
    ed = ((gd.double().cpu() - gd64).norm() / gd64.norm()).item()
    ev = ((gv.double() - gv_ref.double()).norm() / gv_ref.norm()).item()
    print(f"[points mask_loss] P={P} loss={loss.item():.6f} (f64 {loss64.item():.6f}) |dL/dd| rel={ed:.2e} "
          f"|dL/dtemplate| rel={ev:.2e}")
    assert el < 1e-4 and ed < 1e-2 and ev < 1e-2 and gv.abs().sum() > 0
