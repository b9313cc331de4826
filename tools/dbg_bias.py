"""Systematic (signed) relative error of the training GEMM chain vs float64: projection coefficient <ours, true>/<true, true> - 1."""
import os, sys, torch
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from recmv_b200 import ops, synth, testing
from recmv_b200.model import getTmpSdf
dev = "cuda:0"
def proj(a, b):
    a, b = a.double().flatten(), b.double().flatten()
    return float((a @ b) / (b @ b) - 1.0)
for pseed in (None, 101):
    net = testing.build_sdf(getTmpSdf, seed=0, perturb_seed=pseed).to(dev)
    x = (torch.rand((4096, 3), generator=synth.generator(3)) * 1.4 - 0.7).to(dev)
    Ws, bs = [], []
    for l in range(9):
        lin = getattr(net, f"lin{l}")
        Ws.append((lin.weight_v * (lin.weight_g / lin.weight_v.norm(dim=1, keepdim=True))).detach())
        bs.append(lin.bias.detach())
    pe_w = [1.0] * 12
    xd = x.double().requires_grad_(True)
    sdf64, feat64 = ops._sdf_composite(xd, [w.double() for w in Ws], [b.double() for b in bs], pe_w)
    (g64,) = torch.autograd.grad(sdf64.sum(), xd)
    xi = x.clone().requires_grad_(True)
    sdf, feat = ops.SdfMlpTrainFunction.apply(xi, pe_w, None, None, *Ws, *bs)
    (g,) = torch.autograd.grad(sdf.sum(), xi)
    print(f"net {pseed} training Function: forward sdf proj {proj(sdf, sdf64):+.2e} feat {proj(feat, feat64):+.2e}  "
          f"grad proj {proj(g, g64):+.2e}  grad max err {float((g.double() - g64).abs().max() / g64.abs().max()):.2e}")
    xi = x.clone().requires_grad_(True)
    s32, _ = ops._sdf_composite(xi, Ws, bs, pe_w)
    (g32,) = torch.autograd.grad(s32.sum(), xi)
    print(f"net {pseed} torch fp32: forward proj {proj(s32, sdf64):+.2e} grad proj {proj(g32, g64):+.2e}")
    # single GEMMs on operand planes (activations / cotangents scaled 64, weights 1024): mode 4 = forward, 0 = backward-data
    P = 4096
    g = synth.generator(9)
    def act_planes(t, cols):
        return ops.split_planes(t, t.shape[0], cols, 64.0)
    X = torch.randn((P, 512), generator=g).abs().to(dev) * 0.1
    W = Ws[5]
    Y = torch.empty((P, 512), device=dev)
    ops.mlp_layer_planes(act_planes(X, 512), ops.weight_planes(W), P, 512, 512, 4, Y)
    print("  fwd layer (positive acts) proj", f"{proj(Y, X.double() @ W.double().T):+.2e}")
    G = torch.randn((P, 512), generator=g).to(dev)
    D = torch.empty((P, 512), device=dev)
    ops.mlp_layer_planes(act_planes(G, 512), ops.weight_planes(W, transpose=True), P, 512, 512, 0, D)
    print("  bwd-data layer (signed cotangents) proj", f"{proj(D, G.double() @ W.double()):+.2e}")
    ops.mlp_layer_planes(act_planes(G, 512), ops.weight_planes(W), P, 512, 512, 4, Y)
    print("  fwd layer (signed tangents) proj", f"{proj(Y, G.double() @ W.double().T):+.2e}")
    # K = 39 (1 block), K = 257 (5 blocks), weight gradient (32-block chunks), inference engine
    X0 = torch.randn((P, 64), generator=g).to(dev); W0 = Ws[0]
    Y0 = torch.empty((P, 512), device=dev)
    ops.mlp_layer_planes(act_planes(X0, 39), ops.weight_planes(W0), P, 512, 39, 4, Y0)
    print("  fwd layer K=39 proj", f"{proj(Y0, X0[:, :39].double() @ W0.double().T):+.2e}")
    G8 = torch.randn((P, 264), generator=g).to(dev); W8 = Ws[8]
    ops.mlp_layer_planes(act_planes(G8, 257), ops.weight_planes(W8, transpose=True), P, 512, 257, 0, D)
    print("  bwd-data K=257 proj", f"{proj(D, G8[:, :257].double() @ W8.double()):+.2e}")
    for Pw in (2048, 4096, 65536):
        Gw = torch.randn((Pw, 512), generator=g).to(dev); Xw = (torch.randn((Pw, 512), generator=g).abs() * 0.1).to(dev)
        dW = ops.mlp_wgrad_planes(act_planes(Gw, 512), act_planes(Xw, 512), Pw, 512, 512)
        print(f"  weight gradient P={Pw} (signed x positive) proj", f"{proj(dW, Gw.double().T @ Xw.double()):+.2e}")
        Xs = torch.randn((Pw, 512), generator=g).to(dev)
        dW = ops.mlp_wgrad_planes(act_planes(Gw, 512), act_planes(Xs, 512), Pw, 512, 512)
        print(f"  weight gradient P={Pw} (signed x signed) proj", f"{proj(dW, Gw.double().T @ Xs.double()):+.2e}")
    with torch.no_grad():
        y = net(x, None)
    print("  inference engine: sdf proj", f"{proj(y, sdf64):+.2e}", "feat proj", f"{proj(net.rendcond, feat64):+.2e}")
