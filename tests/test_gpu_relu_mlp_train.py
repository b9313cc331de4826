"""The ReLU networks' training Functions (ops.TranslatorTrainFunction, ops.RenderNetTrainFunction) in each backward
branch, end to end through the split of the input-row gradient dX0 into per-argument gradients:
  * the colour network's create_graph input gradient (inside ops.input_grad_only()) against float64 autograd of the same
    network given the Function's own ReLU masks, and a second backward through it;
  * the colour network's create_graph composite (outside input_grad_only()) against the all-torch module;
  * the translator's [N, V, 3] call form in all three branches.
Metric: merr of test_gpu_plane_gemm.py, max |a - b| / max |b| per tensor.  A ReLU network's gradient is discontinuous where
a pre-activation crosses zero, so float64 runs with the masks the Function saved (test_gpu_plane_gemm.py's
_plain_f64_given_our_masks); those may differ from float64's own masks only where |z| < 5e-6."""
import pytest
import torch

from recmv_b200 import ops, synth, testing
import recmv_b200.model as M
from recmv_b200.model.Embedder import ratio_to_weights
from test_gpu_plane_gemm import _plain_f64_given_our_masks, merr

DEV = "cuda:0"
# Bounds measured on an H100 80GB HBM3 (700 W power limit), maximum over every tensor of the file, set about 3x above:
#   against float64 given our masks   4.3e-6 (translator first order lin0.weight; colour input gradient 2.1e-6)
#   composite against all-torch       1.7e-6 (colour lin1.weight_v; translator 1.5e-6)
#   colour composite, tanh'' terms     median row 2.2e-7, 2 of 4099 rows off by > 1e-4 (worst 3.8e-3); biases 1.7e-3
F64_BOUND = 1.5e-5
COMPOSITE_BOUND = 5e-6


@pytest.fixture(autouse=True)
def _no_aborted_launch():
    yield
    if not torch.cuda.is_available():
        return
    torch.cuda.synchronize()
    ops.check_async_errors()


def test_row_widths_are_derived_from_the_layout():
    assert ops.TranslatorTrainFunction.row_width == 168          # [PE6 39 | cond 128] -> 167, padded to 4
    assert ops.RenderNetTrainFunction.row_width == 292           # [p 3 | PE4 27 | n 3 | feat 256] -> 289, padded to 4


def _masks(out, n_in, n=5):
    """The layer inputs [X0, X1, ...] the training Function saved for its output `out` (or a view of it): acts[l + 1] > 0
    are its ReLU masks.  The Function saves (row inputs, Ws, bs, layer inputs, operand planes)."""
    node = out.grad_fn
    while not type(node).__name__.endswith("TrainFunctionBackward"):
        node = node.next_functions[0][0]
    return node.saved_tensors[n_in + 2 * n:n_in + 3 * n]


def _param_grads(mod):
    return [(n, p.grad) for n, p in sorted(mod.named_parameters())]


def _compare(tag, pairs, bound):
    """pairs: (name, ours, reference); both None or both tensors, compared with merr."""
    errs = {}
    for name, a, b in pairs:
        assert (a is None) == (b is None), (tag, name, a is None)
        if a is not None:
            errs[name] = merr(a, b)
    print(f"{tag}: " + ", ".join(f"{k} {v:.1e}" for k, v in errs.items()))
    assert max(errs.values()) < bound, (tag, errs)


def _colour_inputs(R=4099):
    g = synth.generator(31)
    pts = torch.rand((R, 3), generator=g) * 1.2 - 0.6
    nrm = torch.nn.functional.normalize(torch.randn((R, 3), generator=g), dim=1)
    vd = torch.nn.functional.normalize(torch.randn((R, 3), generator=g), dim=1)
    ft = torch.randn((R, 256), generator=g) * 0.5
    cot = torch.randn((R, 3), generator=g) / R
    qs = [torch.randn(t.shape, generator=g) for t in (pts, nrm, vd, ft)]
    return [t.to(DEV) for t in (pts, nrm, vd, ft)], cot.to(DEV), [q.to(DEV) for q in qs]


def _colour_net():
    torch.manual_seed(2)
    rn = M.RenderingNetwork_view_norm(256, d_in=9, d_out=3, dims=[512] * 4, mode="idr", weight_norm=True,
                                      multires_v=4, multires_n=0)
    return testing.perturb_module(rn, 303).to(DEV)


@pytest.mark.gpu
def test_colour_create_graph_input_gradient_matches_fp64_given_our_masks():
    """dp, dn, dv, df of RenderNetTrainFunction's create_graph input-gradient branch, and a second backward through them:
    into the weights and (through the PE's second derivative) the view directions.  Given the masks, the input gradient
    depends on no bias and on neither points, normals nor features."""
    rn = _colour_net()
    Ws, bs = rn.effective_weights()
    Wl = [w.detach().clone().requires_grad_(True) for w in Ws]
    bl = [b.detach().clone().requires_grad_(True) for b in bs]
    ins0, cot, qs = _colour_inputs()
    pe_w = ratio_to_weights(4, 0.8)
    ins = [t.clone().requires_grad_(True) for t in ins0]
    out = ops.RenderNetTrainFunction.apply(*ins, pe_w, *Wl, *bl)
    acts = _masks(out, 4)
    with ops.input_grad_only():
        grads = torch.autograd.grad(out, ins, cot, create_graph=True)
    assert ops.RenderNetTrainFunction.last_backward == "fused-tc (create_graph, input gradient)"
    sum((gr * q).sum() for gr, q in zip(grads, qs)).backward()

    ind = [t.double().requires_grad_(True) for t in ins0]
    Wd = [w.detach().double().requires_grad_(True) for w in Ws]
    bd = [b.detach().double().requires_grad_(True) for b in bs]
    Xd = torch.cat([ind[0], ops._pe_torch(ind[2], pe_w, 4), ind[1], ind[3]], 1)
    h, flips, amb = _plain_f64_given_our_masks(Xd, Wd, bd, acts)
    assert amb == 0, (flips, amb)
    g64 = torch.autograd.grad(h, ind, cot.double(), create_graph=True)
    sum((gr * q.double()).sum() for gr, q in zip(g64, qs)).backward()
    names = ("dp", "dn", "dv", "df")
    pairs = [(k, a, b) for k, a, b in zip(names, grads, g64)]
    pairs += [(f"{k}.grad", a.grad, b.grad) for k, a, b in zip(("points", "normals", "view_dirs", "feats"), ins, ind)]
    pairs += [(f"W{l}", Wl[l].grad, Wd[l].grad) for l in range(5)] + [(f"b{l}", bl[l].grad, bd[l].grad) for l in range(5)]
    assert ins[2].grad is not None and all(t.grad is None for t in (ins[0], ins[1], ins[3]))
    _compare(f"colour input gradient ({flips} mask flips)", pairs, F64_BOUND)


@pytest.mark.gpu
def test_colour_create_graph_composite_matches_the_all_torch_module():
    """Outside input_grad_only() the parameters may want gradients with a graph: the colour network's backward
    differentiates its torch composite, which must agree with the all-torch module (train_fused = False) on the same
    inputs, through a second backward into every parameter and input."""
    rn = _colour_net()
    ins0, cot, qs = _colour_inputs()

    def run(fused):
        rn.train_fused = fused
        rn.zero_grad(set_to_none=True)
        ins = [t.clone().requires_grad_(True) for t in ins0]
        col = rn(*ins, {"renderRatio": 0.8})
        grads = torch.autograd.grad(col, ins, cot, create_graph=True)
        path, label = rn.last_path, ops.RenderNetTrainFunction.last_backward
        sum((gr * q).sum() for gr, q in zip(grads, qs)).backward()
        return path, label, [gr.detach() for gr in grads], [t.grad for t in ins], _param_grads(rn)
    path, label, g1, i1, p1 = run(True)
    assert path == "fused-train" and label == "autograd-composite (create_graph)"
    path, _, g2, i2, p2 = run(False)
    rn.train_fused = True
    assert path == "autograd-composite"
    # The composite's own terms: dp, dn, dv, df and the second backward into the weights and (through the PE) the view
    # directions.
    pairs = [(k, a, b) for k, a, b in zip(("dp", "dn", "dv", "df"), g1, g2)] + [("view_dirs.grad", i1[2], i2[2])]
    pairs += [(n, a, b) for (n, a), (_, b) in zip(p1, p2) if not n.endswith("bias")]
    _compare("colour composite vs all-torch", pairs, COMPOSITE_BOUND)
    # What the second backward sends to points, normals, features and biases comes only through tanh'' and the first-order
    # backward of the forward that produced the colour: fused here, torch there.  A unit within fp32 noise of zero can
    # flip its ReLU mask between the two and move that row's entries, so these are compared per row and per tensor.
    for k, a, b in zip(("points", "normals", "feats"), (i1[0], i1[1], i1[3]), (i2[0], i2[1], i2[3])):
        e = (a - b).abs().amax(1) / b.abs().max()
        print(f"colour composite {k}.grad: median row {float(e.median()):.1e}, rows off by > 1e-4: {int((e > 1e-4).sum())}"
              f" of {e.numel()}, worst {float(e.max()):.1e}")
        assert float(e.median()) < 1e-6 and int((e > 1e-4).sum()) <= 6, k
    biases = {n: merr(a, b) for (n, a), (_, b) in zip(p1, p2) if n.endswith("bias")}
    print("colour composite biases: " + ", ".join(f"{k} {v:.1e}" for k, v in biases.items()))
    assert max(biases.values()) < 5e-3, biases


@pytest.mark.gpu
@pytest.mark.parametrize("branch", ["first-order", "input gradient", "composite"])
def test_translator_nv3_form_in_each_branch(branch):
    """MLPTranslator called with ps [N, V, 3] and one condition per frame (no batch_inds): first order and the create_graph
    input gradient against float64 given the Function's own masks; the create_graph composite against the all-torch
    module.  The create_graph branches are followed by a second backward."""
    torch.manual_seed(1)
    tr = testing.perturb_module(M.MLPTranslator(128, 6), 202, scale=0.5).to(DEV)
    N, V = 3, 1500
    g = synth.generator(41)
    p0 = (torch.rand((N, V, 3), generator=g) * 1.2 - 0.6).to(DEV)
    c0 = (torch.randn((N, 128), generator=g) * 0.3).to(DEV)
    cot = (torch.randn((N, V, 3), generator=g) / (N * V)).to(DEV)
    qs = [torch.randn((N, V, 3), generator=g).to(DEV), torch.randn((N, 128), generator=g).to(DEV)]
    ratio = {"deformerRatio": 0.6}

    def run(create_graph, fused=True):
        tr.train_fused = fused
        tr.zero_grad(set_to_none=True)
        p, c = p0.clone().requires_grad_(True), c0.clone().requires_grad_(True)
        out = tr(p, c, None, ratio=ratio, offset_type="nv3")
        assert tr.last_path == ("fused-train" if fused else "autograd-composite")
        acts = _masks(tr.offset["nv3"], 3) if fused else None
        if not create_graph:
            (out * cot).sum().backward()
            return acts, None, [p.grad, c.grad], _param_grads(tr)
        grads = torch.autograd.grad(out, [p, c], cot, create_graph=True)
        sum((gr * q).sum() for gr, q in zip(grads, qs)).backward()
        return acts, [gr.detach() for gr in grads], [p.grad, c.grad], _param_grads(tr)

    if branch == "composite":
        _, g1, i1, p1 = run(True)
        assert ops.TranslatorTrainFunction.last_backward == "autograd-composite (create_graph)"
        _, g2, i2, p2 = run(True, fused=False)
        tr.train_fused = True
        pairs = [("dp", g1[0], g2[0]), ("dconds", g1[1], g2[1]), ("ps.grad", i1[0], i2[0]), ("conds.grad", i1[1], i2[1])]
        pairs += [(n, a, b) for (n, a), (_, b) in zip(p1, p2)]
        _compare("translator [N,V,3] composite vs all-torch", pairs, COMPOSITE_BOUND)
        return
    if branch == "first-order":
        acts, _, i1, p1 = run(False)
        assert ops.TranslatorTrainFunction.last_backward == "fused-tc"
    else:
        with ops.input_grad_only():
            acts, g1, i1, p1 = run(True)
        assert ops.TranslatorTrainFunction.last_backward == "fused-tc (create_graph, input gradient)"
    pd, cd = p0.double().requires_grad_(True), c0.double().requires_grad_(True)
    Wd = [getattr(tr, f"lin{l}").weight.detach().double().requires_grad_(True) for l in range(5)]
    bd = [getattr(tr, f"lin{l}").bias.detach().double().requires_grad_(True) for l in range(5)]
    frame = torch.arange(N, device=DEV).repeat_interleave(V)
    Xd = torch.cat([ops._pe_torch(pd.reshape(-1, 3), ratio_to_weights(6, 0.6), 6), cd[frame]], 1)
    h, flips, amb = _plain_f64_given_our_masks(Xd, Wd, bd, acts)
    assert amb == 0, (flips, amb)
    out64 = pd + h.view(N, V, 3)
    pairs = []
    if branch == "first-order":
        (out64 * cot.double()).sum().backward()
    else:
        g64 = torch.autograd.grad(out64, [pd, cd], cot.double(), create_graph=True)
        sum((gr * q.double()).sum() for gr, q in zip(g64, qs)).backward()
        pairs += [("dp", g1[0], g64[0]), ("dconds", g1[1], g64[1])]
    pairs += [("ps.grad", i1[0], pd.grad), ("conds.grad", i1[1], cd.grad)]
    pairs += [(n, a, b.grad) for (n, a), b in zip(p1, [t for l in range(5) for t in (bd[l], Wd[l])])]  # lin0.bias, lin0.weight, ...
    _compare(f"translator [N,V,3] {branch} ({flips} mask flips)", pairs, F64_BOUND)
