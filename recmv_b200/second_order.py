"""Second order on the tensor-core GEMMs (SURVEY 8f row 4): the input gradient of the three MLPs as a DIFFERENTIABLE op.

The reference differentiates its networks twice on every training step:
  * eikonal loss        -- `ImplicitNetwork.gradient` (model/network.py:121-133: autograd.grad(y, x, create_graph=True)),
                           then ((|grad| - 1)^2).mean().backward()        (engineer/networks/OptimGarmentNetwork.py:1108-1118)
  * deformed normals    -- utils.compute_deformed_normals in the train phase (utils/utils.py:198-230)
  * deformation regulariser -- utils.compute_Jacobian(ps, defVs, True, True) of the translator, singular values, log, robust
                           error                                          (OptimGarmentNetwork.py:1135-1154)

`ops.SdfMlpTrainFunction.backward` / `ops.TranslatorTrainFunction.backward` / `ops.RenderNetTrainFunction.backward` called
with create_graph=True land here when only INPUT gradients are requested (the three call sites above): the reverse chain
is itself an autograd Function whose backward is

    upward   : the network's tangent (JVP) pass  tz_l = tu_l W_l^T,  tu_{l+1} = act'(z_l) * tz_l       (9 layer GEMMs)
    local    : zb_l = act''(z_l) * u_{l+1} * tz_l  = 100 (1 - s_l) h_{l+1} tz_l   for softplus_100 (0 for ReLU)
    downward : an ordinary backward-data pass that picks zb_l up at every layer                       (8 layer GEMMs)
    weights  : dW_l = h_{l+1}^T tu_l + zb_l^T a_l,  db_l = sum zb_l

with h_{l+1} the first-order cotangent at z_l.  Everything heavy is a 3xfp16 wgmma GEMM on the operand-plane kernels of
csrc/gemm3_tma.cu.  Each network's reverse chain is its first-order path's own (ops.sdf_reverse_chain,
ops.plain_reverse_chain).  In the SDF network's backward every GEMM is followed by one element-wise launch that also writes
the next GEMM's planes; the ReLU networks' tangent pass applies the ReLU mask in the GEMM epilogue and needs no such
launch.  The positional encoding's own VJP is a torch graph (so its second derivative comes from autograd).  A request
that ALSO wants parameter gradients with a graph (loss.backward(create_graph=True)) still takes the torch-composite
fallback."""
import torch

from . import ops
from .ops import _INV_SQRT2, _pad8, _plane_pair, grad_dyn_scale, mlp_layer_planes, pe_backward, split_planes


def pe_vjp_torch(x, u, pe_w, bands):
    """(d PE(x) / d x)^T u as a torch graph: x [P,3], u [P, >= 3 + 6 bands] -> [P,3]."""
    out = u[:, 0:3]
    f = 1.0
    for k in range(bands):
        c = 3 + 6 * k
        out = out + (pe_w[2 * k] * f) * torch.cos(x * f) * u[:, c:c + 3] - (pe_w[2 * k + 1] * f) * torch.sin(x * f) * u[:, c + 3:c + 6]
        f *= 2.0
    return out


class SdfMlpPeGradFunction(torch.autograd.Function):
    """u0 [P,39] = d(g_sdf . sdf + g_feat . feat) / d PE  of ImplicitNetwork (both PE entry points: layer 0 and the skip
    of layer 4), from the activations the training forward saved.  Differentiable in g, the weights and (through the
    activations) x -- see the module docstring for the backward."""

    @staticmethod
    def forward(ctx, x, g_sdf, g_feat, pe_w, *rest):
        act, Ws, xplanes = rest[:9], rest[9:18], rest[27:]
        dyn, G, GP, dpe0, dpe4 = ops.sdf_reverse_chain(g_sdf, g_feat, act, Ws)
        ctx.pe_w = [float(w) for w in pe_w]
        ctx.dims = ([w.shape[0] for w in Ws], [w.shape[1] for w in Ws])
        ctx.save_for_backward(x, dyn, *act, *Ws, *G, *[t for pair in GP for t in pair], *xplanes)
        return (dpe0 + dpe4)[:, :39].contiguous()

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, q):
        """On the TMA-fed plane GEMMs (csrc/gemm3_tma.cu): every layer is ONE GEMM launch plus ONE element-wise launch that
        also writes the next GEMM's operand planes."""
        saved = ctx.saved_tensors
        x, dyn = saved[0], saved[1]
        act, Ws, G = saved[2:11], saved[11:20], saved[20:29]
        GPl, XPl = saved[29:47], saved[47:65]
        outs, ins = ctx.dims
        need = ctx.needs_input_grad
        need_x, need_g = need[0], need[1] or need[2]
        need_w = any(need[13:31])
        P, dev = x.shape[0], x.device
        dq = grad_dyn_scale(q)
        inv_dq = 1.0 / dq
        sc = [_INV_SQRT2 if l == 4 else 1.0 for l in range(9)]
        # ---- upward: tangent pass with tangent of PE = q (scaled into [1,2) by dq; everything below is linear in it) ----
        U = [torch.zeros((P, 64), dtype=torch.float32, device=dev)] + \
            [torch.zeros((P, 512), dtype=torch.float32, device=dev) for _ in range(8)]
        U[0][:, :39] = q * dq
        U[4][:, 473:] = U[0][:, :39]
        up = up0 = split_planes(U[0], P, 39, 64.0, ldp=64)
        UP = [up0] + [None] * 8
        inj = [None] * 8
        tz = None
        for l in range(9):
            o = outs[l]
            tz = torch.empty((P, 512 if l < 8 else 264), dtype=torch.float32, device=dev)
            mlp_layer_planes(up, ops.weight_planes(Ws[l]), P, o, ins[l], 4, tz, scale=sc[l])
            if l < 8:
                un = _plane_pair(P, 512, dev, zero=True)
                inj[l] = torch.zeros((P, 512), dtype=torch.float32, device=dev)
                ops.softplus_tangent_planes(tz, act[l + 1], G[l], o, U[l + 1], un, inj[l])
                if l == 3:      # layer 4 reads [tangent of a_4 (473) | tangent of PE (39)]
                    un[0][:, 473:] = up0[0][:, :39]
                    un[1][:, 473:] = up0[1][:, :39]
                up = un
                UP[l + 1] = un
        g_bar = tz[:, :257] * inv_dq if need_g else None
        # ---- downward: backward-data pass that collects the local terms ----
        dx = None
        dW, db = [None] * 9, [None] * 9
        if need_x or need_w:
            dyn2 = grad_dyn_scale(*inj)
            Zb = [None] * 8
            Zb[7] = inj[7]
            zp = split_planes(Zb[7], P, 512, 64.0, scale_dev=dyn2, ldp=512)
            ZP = [None] * 8
            ZP[7] = zp
            dpe4 = torch.zeros((P, 40), dtype=torch.float32, device=dev)
            for l in range(7, 0, -1):
                Zb[l - 1] = torch.zeros((P, 512), dtype=torch.float32, device=dev)
                mlp_layer_planes(zp, ops.weight_planes(Ws[l], transpose=True), P, ins[l], outs[l], 1, Zb[l - 1],
                                 saved_input=act[l], scale=sc[l], dyn=dyn2, a_has_dyn=True, split=473 if l == 4 else 0,
                                 Y2=dpe4 if l == 4 else None)
                zp = _plane_pair(P, 512, dev, zero=True)
                ops.add_split_planes(Zb[l - 1], inj[l - 1], outs[l - 1], zp, 64.0, dyn2)
                ZP[l - 1] = zp
            if need_x:
                dpe0 = torch.zeros((P, 40), dtype=torch.float32, device=dev)
                mlp_layer_planes(zp, ops.weight_planes(Ws[0], transpose=True), P, ins[0], outs[0], 0, dpe0,
                                 dyn=dyn2, a_has_dyn=True)
                dx = pe_backward(x, dpe0, dpe4, ctx.pe_w, 6) * inv_dq
            if need_w:
                # both outer products straight from the planes the passes wrote (recmv_mlp_wgrad_planes)
                for l in range(9):
                    w1 = ops.mlp_wgrad_planes((GPl[2 * l], GPl[2 * l + 1]), UP[l], P, outs[l], ins[l], sc[l], dyn)
                    if l < 8:
                        w2, b2 = ops.mlp_wgrad_planes(ZP[l], (XPl[2 * l], XPl[2 * l + 1]), P, outs[l], ins[l], sc[l], dyn2,
                                                      want_bias=True)
                        w1 = w1 + w2
                        db[l] = b2 * inv_dq
                    dW[l] = w1 * inv_dq
        g_sdf_bar = g_bar[:, 0:1].contiguous() if (need[1] and g_bar is not None) else None
        g_feat_bar = g_bar[:, 1:257].contiguous() if (need[2] and g_bar is not None) else None
        return (dx, g_sdf_bar, g_feat_bar, None, *([None] * 9), *dW, *db, *([None] * (len(need) - 31)))


def sdf_input_grad(x, g_sdf, g_feat, pe_w, act, Ws, bs, xplanes):
    """dx of ImplicitNetwork as a twice-differentiable expression (the create_graph=True branch of
    ops.SdfMlpTrainFunction.backward).  xplanes: the forward's 18 layer-input operand planes (flat hi, lo list)."""
    u0 = SdfMlpPeGradFunction.apply(x, g_sdf, g_feat, pe_w, *act, *Ws, *bs, *xplanes)
    return pe_vjp_torch(x, u0, pe_w, 6)


class PlainMlpInputGradFunction(torch.autograd.Function):
    """dX0 [P, in_0] = (d out / d X0)^T g_out of a ReLU MLP (translator, colour network) from the saved layer inputs;
    differentiable in g_out and the weights (ReLU'' = 0: no dependence on X0 itself, no bias gradient)."""

    @staticmethod
    def forward(ctx, g_out, n, *rest):
        acts, Ws = rest[:n], rest[n:2 * n]
        dyn, GP, dX0 = ops.plain_reverse_chain(g_out, Ws, acts)
        ctx.n = n
        ctx.save_for_backward(dyn, *acts, *Ws, *[t for pair in GP for t in pair])
        return dX0[:, :Ws[0].shape[1]]

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, q):
        """Tangent pass on the plane GEMMs: U_{l+1} = (U_l W_l^T) * [a_{l+1} > 0], one backward-data launch with the ReLU'
        epilogue per layer (the [out][in] weight planes make it the forward product), then dW_l = h_{l+1}^T U_l from the
        cotangent planes the forward saved and the tangent planes."""
        n = ctx.n
        saved = ctx.saved_tensors
        dyn = saved[0]
        acts, Ws, GPl = saved[1:1 + n], saved[1 + n:1 + 2 * n], saved[1 + 2 * n:]
        need = ctx.needs_input_grad
        P, dev = q.shape[0], q.device
        dq = grad_dyn_scale(q)
        inv_dq = 1.0 / dq
        i0 = Ws[0].shape[1]
        UP = [split_planes(q * dq, P, i0, 64.0, ldp=_pad8(i0))]
        for l in range(n - 1):
            o, i = Ws[l].shape
            un = _plane_pair(P, _pad8(o), dev)
            mlp_layer_planes(UP[l], ops.weight_planes(Ws[l]), P, o, i, 2, torch.empty((P, o), dtype=torch.float32, device=dev),
                             saved_input=acts[l + 1], y_planes=un)
            UP.append(un)
        g_bar = None
        if need[0]:
            o, i = Ws[-1].shape
            tz = torch.empty((P, ((o + 3) // 4) * 4), dtype=torch.float32, device=dev)
            mlp_layer_planes(UP[-1], ops.weight_planes(Ws[-1]), P, o, i, 0, tz)
            g_bar = tz[:, :o] * inv_dq
        dW = [None] * n
        if any(need[2 + n:2 + 2 * n]):
            dW = [ops.mlp_wgrad_planes((GPl[2 * l], GPl[2 * l + 1]), UP[l], P, Ws[l].shape[0], Ws[l].shape[1], 1.0, dyn) * inv_dq
                  for l in range(n)]
        return (g_bar, None, *([None] * n), *dW)
