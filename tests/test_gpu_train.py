"""GPU parity of the TRAINING path of the three networks: the forward that saves the layer inputs and the tensor-core
backward GEMMs (csrc/gemm3_tma.cu) behind `loss.backward()`, against
  * the gradients torch autograd produces through the REFERENCE's own classes (fp32 = the reference's numbers,
    fp64 = ground truth), tests/golden/{sdf_bwd_*,translator_bwd,rendernet_bwd}.npz from tests/golden/make_golden_r2.py;
  * fp64 matmuls for the weight gradient on the operand planes at ragged shapes.
Metric: max |a - b| / max |b| per tensor (a gradient tensor's entries span decades; its scale is its largest entry).
Bound 3e-5 against the fp64 truth (the reference's own fp32 autograd sits 2e-7 .. 9e-6 from it in the same metric)."""
import numpy as np
import pytest
import torch

from conftest import load_golden
from recmv_b200 import _lib, ops, synth, testing
from recmv_b200.model import getTmpSdf

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


@pytest.fixture(autouse=True)
def _no_aborted_launch():
    yield
    torch.cuda.synchronize()
    ops.check_async_errors()


def cotangents(P, nfeat, seed):      # tests/golden/make_golden_r2.py
    g = synth.generator(seed)
    mag = torch.exp(torch.randn((P, 1), generator=g) * 1.0) / P
    c0 = torch.randn((P, 1), generator=g) * mag
    c1 = torch.randn((P, nfeat), generator=g) * mag * 0.1
    return c0, c1


def merr(a, b):
    a = torch.as_tensor(a, dtype=torch.float64).detach().cpu()
    b = torch.as_tensor(b, dtype=torch.float64).detach().cpu()
    return float((a - b).abs().max() / b.abs().max().clamp_min(1e-300))


@pytest.mark.parametrize("tag", ["geo", "trained"])
def test_loss_backward_matches_reference_autograd(tag):
    g = load_golden(f"sdf_bwd_{tag}.npz")
    x0 = torch.from_numpy(load_golden(f"sdf_c1_{tag}.npz")["x"])[:2048]
    net = testing.build_sdf(getTmpSdf, seed=0, perturb_seed=None if tag == "geo" else 101).to(DEV)
    c0, c1 = cotangents(2048, 256, 77)
    x = x0.to(DEV).requires_grad_(True)
    y = net(x, {'sdfRatio': 0.7})
    assert net.last_path == "fused-train"
    loss = (y * c0.to(DEV)).sum() + (net.rendcond * c1.to(DEV)).sum()
    loss.backward()
    assert ops.SdfMlpTrainFunction.last_backward == "fused-tc"
    rows = [("dx", merr(x.grad, g["dx_f64"]), merr(g["dx_f32"], g["dx_f64"]))]
    for l in range(9):
        lin = getattr(net, f"lin{l}")
        rows.append((f"lin{l}.bias", merr(lin.bias.grad, g[f"f64_lin{l}_bias"]), merr(g[f"f32_lin{l}_bias"], g[f"f64_lin{l}_bias"])))
        rows.append((f"lin{l}.weight_g", merr(lin.weight_g.grad, g[f"f64_lin{l}_weight_g"]),
                     merr(g[f"f32_lin{l}_weight_g"], g[f"f64_lin{l}_weight_g"])))
        gv = lin.weight_v.grad
        if f"f64_lin{l}_weight_v_sample" in g:
            for part, ours in (("sample", gv[::16, ::8]), ("rowsum", gv.double().sum(1)), ("colsum", gv.double().sum(0))):
                k = f"lin{l}_weight_v_{part}"
                scale = float(g[f"f64_lin{l}_weight_v_absmax"]) * (1 if part == "sample" else 16)
                e = float((torch.as_tensor(ours).double().cpu() - torch.from_numpy(g["f64_" + k]).double()).abs().max()) / scale
                e_ref = float(np.abs(g["f32_" + k].astype(np.float64) - g["f64_" + k]).max()) / scale
                rows.append((k, e, e_ref))
        else:
            rows.append((f"lin{l}.weight_v", merr(gv, g[f"f64_lin{l}_weight_v"]), merr(g[f"f32_lin{l}_weight_v"], g[f"f64_lin{l}_weight_v"])))
    table = "\n".join(f"{tag}/{n}: |ours-f64| {a:.2e}  |ref32-f64| {b:.2e}" for n, a, b in rows)
    print(table)
    for n, a, b in rows:   # row / column sums of a weight gradient are sums of 512 signed entries: looser relative scale
        assert a < (2e-4 if n.endswith("sum") else 3e-5), table


def test_create_graph_input_gradient_matches_the_all_torch_module():
    """gradient(x) with create_graph=True (network.py:121-133; eikonal term): second-order gradients through the fused
    reverse chain (recmv_b200/second_order.py) agree with the all-torch module (float64 parity: test_gpu_second_order.py)."""
    net = testing.build_sdf(getTmpSdf, seed=0, perturb_seed=101).to(DEV)
    x0 = (torch.rand((512, 3), generator=synth.generator(5)) * 1.2 - 0.6).to(DEV)

    def eikonal(fused):
        net.train_fused = fused
        net.zero_grad()
        x = x0.clone().requires_grad_(True)
        gr = net.gradient(x)
        loss = ((gr.norm(dim=1) - 1) ** 2).mean()
        loss.backward()
        return gr.detach(), [None if p.grad is None else p.grad.clone() for p in net.parameters()], x.grad.clone()
    g1, p1, x1 = eikonal(True)
    assert net.last_path == "fused-train" and "create_graph" in ops.SdfMlpTrainFunction.last_backward
    g2, p2, x2 = eikonal(False)
    assert net.last_path == "autograd-composite"
    assert merr(g1, g2) < 1e-4 and merr(x1, x2) < 2e-3
    for a, b in zip(p1, p2):
        assert (a is None) == (b is None)      # e.g. the last bias: the input gradient does not depend on it
        if a is not None:
            assert merr(a, b) < 2e-3
    net.train_fused = True


def _grad_rows(prefix, named_params, g):
    rows = []
    for name, prm in named_params:
        key = name.replace(".", "_")
        gv = prm.grad
        if f"f64_{key}_sample" in g:
            for part, ours in (("sample", gv[::16, ::8]), ("rowsum", gv.double().sum(1)), ("colsum", gv.double().sum(0))):
                scale = float(g[f"f64_{key}_absmax"]) * (1 if part == "sample" else 16)
                e = float((torch.as_tensor(ours).double().cpu() - torch.from_numpy(g[f"f64_{key}_{part}"]).double()).abs().max()) / scale
                e_ref = float(np.abs(g[f"f32_{key}_{part}"].astype(np.float64) - g[f"f64_{key}_{part}"]).max()) / scale
                rows.append((f"{prefix}{key}_{part}", e, e_ref))
        else:
            rows.append((prefix + key, merr(gv, g["f64_" + key]), merr(g["f32_" + key], g["f64_" + key])))
    return rows


def test_translator_backward_matches_reference_autograd():
    """MLPTranslator (model/Deformer.py:171-206) on the tensor-core training path vs the reference class's autograd."""
    import recmv_b200.model as M
    g = load_golden("translator_bwd.npz")
    gi = load_golden("translator.npz")
    torch.manual_seed(1)
    tr = testing.perturb_module(M.MLPTranslator(128, 6), 202, scale=0.5).to(DEV)
    p = torch.from_numpy(gi["p"]).to(DEV).requires_grad_(True)
    conds = torch.from_numpy(gi["conds"]).to(DEV).requires_grad_(True)
    binds = torch.from_numpy(gi["batch_inds"]).to(DEV)
    out = tr(p, conds, binds, ratio={"deformerRatio": 0.6}, offset_type="body")
    assert tr.last_path == "fused-train" and merr(out, gi["out"]) < 2e-5
    (out * torch.from_numpy(g["cot"]).to(DEV)).sum().backward()
    assert ops.TranslatorTrainFunction.last_backward == "fused-tc"
    rows = [("dp", merr(p.grad, g["dp_f64"]), merr(g["dp_f32"], g["dp_f64"])),
            ("dconds", merr(conds.grad, g["dconds_f64"]), merr(g["dconds_f32"], g["dconds_f64"]))]
    rows += _grad_rows("", sorted(tr.named_parameters()), g)
    table = "\n".join(f"translator/{n}: |ours-f64| {a:.2e}  |ref32-f64| {b:.2e}" for n, a, b in rows)
    print(table)
    # A ReLU network's gradient is discontinuous where a pre-activation crosses zero: this fixture has units with
    # |z| down to 2.5e-8 (layer 1), so ANY fp32-level difference in the forward flips a few of 4 M masks and moves single
    # gradient entries by ~1e-3 of the tensor's scale.  Two exact statements instead of one fuzzy bound:
    #  (1) our masks differ from the float64 masks only at such ambiguous units;
    #  (2) given OUR masks, every gradient agrees with float64 autograd to 1e-4 of its scale.
    from recmv_b200.model.Embedder import ratio_to_weights
    Ws = [getattr(tr, f"lin{l}").weight.detach() for l in range(5)]
    bs = [getattr(tr, f"lin{l}").bias.detach() for l in range(5)]
    x0 = torch.cat([tr.embed_fn(p.detach(), ratio_to_weights(6, 0.6)), conds.detach()[binds]], 1)
    X0 = torch.zeros((x0.shape[0], 168), device=DEV)
    X0[:, :167] = x0
    _, acts, _ = ops._plain_mlp_forward(X0, Ws, bs)                      # the same launches the Function's forward makes
    pd, cd = p.detach().double().requires_grad_(True), conds.detach().double().requires_grad_(True)
    Wd = [w.double().requires_grad_(True) for w in Ws]
    bd = [b.double().requires_grad_(True) for b in bs]
    h = torch.cat([tr.embed_fn(pd, ratio_to_weights(6, 0.6)), cd[binds]], 1)
    flips = amb = 0
    for l in range(5):
        z = torch.nn.functional.linear(h, Wd[l], bd[l])
        if l < 4:
            ours = acts[l + 1] > 0
            diff = ours != (z > 0)
            flips += int(diff.sum())
            amb += int((diff & (z.abs() > 5e-6)).sum())
            h = z * ours.double()
        else:
            h = z
    assert amb == 0 and flips < 200, (flips, amb)                     # (1)
    ((pd + h) * torch.from_numpy(g["cot"]).to(DEV).double()).sum().backward()
    checks = [("dp", p.grad, pd.grad), ("dconds", conds.grad, cd.grad)]
    checks += [(f"lin{l}.weight", getattr(tr, f"lin{l}").weight.grad, Wd[l].grad) for l in range(5)]
    checks += [(f"lin{l}.bias", getattr(tr, f"lin{l}").bias.grad, bd[l].grad) for l in range(5)]
    errs = {n: merr(a, b) for n, a, b in checks}
    print(f"translator: {flips} mask flips against float64 (all at |z| < 5e-6); with our masks: "
          + ", ".join(f"{n} {e:.1e}" for n, e in errs.items()))
    assert max(errs.values()) < 1e-4, errs                            # (2)  (measured 3e-8 .. 4.3e-5)
    for n, a, b in rows:   # tensors no flipped unit feeds (downstream layers, dp) also match the fixture directly
        if n in ("dp",) or n.startswith(("lin2", "lin3", "lin4")):
            assert a < (2e-4 if n.endswith("sum") else 3e-5), table
    # [N, V, 3] call form and second order through the torch fallback
    p2 = torch.from_numpy(gi["p"][:1500]).to(DEV).view(3, 500, 3).requires_grad_(True)
    o2 = tr(p2, conds, None, ratio={"deformerRatio": 0.6}, offset_type="b2")
    gr = torch.autograd.grad(o2.sum(), p2, create_graph=True)[0]
    gr.pow(2).sum().backward()
    assert "create_graph" in ops.TranslatorTrainFunction.last_backward and torch.isfinite(p2.grad).all()


def test_rendernet_backward_matches_reference_autograd():
    """RenderingNetwork_view_norm (model/RenderNet.py:59-96) on the tensor-core training path vs the reference's autograd."""
    import recmv_b200.model as M
    g = dict(load_golden("rendernet_bwd.npz"), **load_golden("rendernet_feats.npz"))
    torch.manual_seed(2)
    rn = M.RenderingNetwork_view_norm(256, d_in=9, d_out=3, dims=[512] * 4, mode="idr", weight_norm=True,
                                      multires_v=4, multires_n=0)
    rn = testing.perturb_module(rn, 303).to(DEV)
    ins = [torch.from_numpy(g[k]).to(DEV).requires_grad_(True) for k in ("points", "normals", "view_dirs", "feats")]
    col = rn(ins[0], ins[1], ins[2], ins[3], {"renderRatio": 0.8})
    assert rn.last_path == "fused-train"
    (col * torch.from_numpy(g["cot"]).to(DEV)).sum().backward()
    assert ops.RenderNetTrainFunction.last_backward == "fused-tc"
    rows = [("dpoints", merr(ins[0].grad, g["dpoints_f64"]), merr(g["dpoints_f32"], g["dpoints_f64"])),
            ("dnormals", merr(ins[1].grad, g["dnormals_f64"]), merr(g["dnormals_f32"], g["dnormals_f64"])),
            ("dview", merr(ins[2].grad, g["dview_f64"]), merr(g["dview_f32"], g["dview_f64"])),
            ("dfeats", merr(ins[3].grad[:, ::8], g["dfeats_f64"]), merr(g["dfeats_f32"], g["dfeats_f64"]))]
    rows += _grad_rows("", sorted(rn.named_parameters()), g)
    table = "\n".join(f"rendernet/{n}: |ours-f64| {a:.2e}  |ref32-f64| {b:.2e}" for n, a, b in rows)
    print(table)
    for n, a, b in rows:
        assert a < (2e-4 if n.endswith("sum") else 3e-5), table


@pytest.mark.parametrize("P,out_dim,in_dim", [(64, 128, 128), (3000, 473, 512), (1, 257, 512), (4097, 512, 39), (70000, 512, 512)])
def test_wgrad_on_planes_matches_fp64(P, out_dim, in_dim):
    """recmv_mlp_wgrad_planes (MN-major operands straight from the row-major planes) and recmv_colsum vs float64."""
    g = synth.generator(40 + P % 7)
    G = (torch.randn((P, 512), generator=g) * torch.exp(torch.randn((P, 1), generator=g)) * 1e-3).to(DEV)
    X = torch.randn((P, 512), generator=g).abs().mul(0.3).to(DEV)
    dyn = ops.grad_dyn_scale(G)
    gp = ops.split_planes(G, P, out_dim, 64.0, scale_dev=dyn, ldp=512)
    xp = ops.split_planes(X, P, in_dim, 64.0, ldp=512)
    dW, db_mma = ops.mlp_wgrad_planes(gp, xp, P, out_dim, in_dim, 0.5, dyn, want_bias=True)
    ref = 0.5 * G[:, :out_dim].double().T @ X[:, :in_dim].double()
    e = merr(dW, ref)
    assert torch.equal(dW, ops.mlp_wgrad_planes(gp, xp, P, out_dim, in_dim, 0.5, dyn))      # deterministic, with or without db
    db = ops.colsum(G, out_dim)
    ref_b = G[:, :out_dim].double().sum(0)
    eb = merr(db, ref_b)
    ebm = merr(db_mma, ref_b)
    print(f"wgrad planes P={P} {out_dim}x{in_dim}: {e:.2e}  colsum {eb:.2e}  bias gradient from the ones tile {ebm:.2e}")
    assert ebm < 5e-6
    assert e < (6e-6 if P > 10000 else 3e-6) and eb < 2e-6      # measured 3.3e-6 at 70 000 samples
