"""ImplicitNetwork / getTmpSdf with the reference's constructor, parameters and forward contract
(model/network.py:27-141), dispatching the forward to the fused sm_100a kernel.

State-dict keys are identical (lin{0..8}.{weight_g,weight_v,bias}) so reference checkpoints load.
Paths:
  * no autograd needed (torch.no_grad(), C2F sweep, convergence checks, inference): ONE fused launch
    (PE + 9 linears + softplus, activations never leave the SM) via recmv_sdf_mlp_fwd;
  * autograd needed: the same math as a torch graph over the module's parameters (twice
    differentiable, as `create_graph=True` callers require -- network.py:121-133).  `last_path`
    records which one ran; nothing falls back silently to a CPU implementation.
"""
import numpy as np
import torch
import torch.nn as nn

from .. import ops
from .Embedder import get_embedder, ratio_to_weights
from .packed import cached_pack


class ImplicitNetwork(nn.Module):
    def __init__(self, feature_vector_size, d_in, d_out, dims, geometric_init=True, bias=1.0,
                 skip_in=(), weight_norm=True, multires=0):
        super().__init__()
        dims = [d_in] + dims + [d_out + feature_vector_size]
        self.d_out = d_out
        self.embed_fn = None
        self.multires = multires
        if multires > 0:
            embed_fn, input_ch = get_embedder(multires)
            self.embed_fn = embed_fn
            dims[0] = input_ch
        self.num_layers = len(dims)
        self.skip_in = skip_in
        self.uses_weight_norm = weight_norm
        for l in range(0, self.num_layers - 1):
            out_dim = dims[l + 1] - dims[0] if l + 1 in self.skip_in else dims[l + 1]
            lin = nn.Linear(dims[l], out_dim)
            if geometric_init:  # network.py:63-78
                if l == self.num_layers - 2:
                    torch.nn.init.normal_(lin.weight, mean=np.sqrt(np.pi) / np.sqrt(dims[l]), std=0.0001)
                    torch.nn.init.constant_(lin.bias, -bias)
                elif multires > 0 and l == 0:
                    torch.nn.init.constant_(lin.bias, 0.0)
                    torch.nn.init.constant_(lin.weight[:, 3:], 0.0)
                    torch.nn.init.normal_(lin.weight[:, :3], 0.0, np.sqrt(2) / np.sqrt(out_dim))
                elif multires > 0 and l in self.skip_in:
                    torch.nn.init.constant_(lin.bias, 0.0)
                    torch.nn.init.normal_(lin.weight, 0.0, np.sqrt(2) / np.sqrt(out_dim))
                    torch.nn.init.constant_(lin.weight[:, -(dims[0] - 3):], 0.0)
                else:
                    torch.nn.init.constant_(lin.bias, 0.0)
                    torch.nn.init.normal_(lin.weight, 0.0, np.sqrt(2) / np.sqrt(out_dim))
            if weight_norm:
                lin = nn.utils.weight_norm(lin)
            setattr(self, "lin" + str(l), lin)
        self.softplus = nn.Softplus(beta=100)
        self.rendcond = None
        self.mlp_mode = None  # None -> ops.DEFAULT_MLP_MODE
        self.train_fused = True   # grad-enabled forwards go through ops.SdfMlpTrainFunction (False: torch graph)
        self.last_path = None
        shapes = [tuple(getattr(self, "lin%d" % l).weight.shape) for l in range(self.num_layers - 1)]
        self._fusable = (shapes == ops.SDF_LAYER_SHAPES and tuple(self.skip_in) == (4,)
                         and multires == 6 and d_out == 1)

    # -- effective weights / packed blob cache ------------------------------------------------
    def effective_weights(self):
        Ws, bs = [], []
        for l in range(self.num_layers - 1):
            lin = getattr(self, "lin%d" % l)
            if self.uses_weight_norm:
                g, v = lin.weight_g, lin.weight_v
                Ws.append(g * v / v.norm(dim=1, keepdim=True))
            else:
                Ws.append(lin.weight)
            bs.append(lin.bias)
        return Ws, bs

    def packed_weights(self):
        return cached_pack(self, lambda: ops.sdf_pack_weights(*self.effective_weights()))

    def _pe_weights(self, ratio):
        ratio = ratio if type(ratio) == float or type(ratio) == int or ratio is None else ratio['sdfRatio']
        return ratio_to_weights(self.multires, ratio)

    # -- forward ----------------------------------------------------------------------------
    def forward(self, input, ratio):
        needs_graph = torch.is_grad_enabled() and (
            input.requires_grad or any(p.requires_grad for p in self.parameters()))
        if self._fusable and input.is_cuda and not needs_graph:
            self.last_path = "fused"
            sdf, feat = ops.sdf_mlp_forward(input.reshape(-1, 3), self.packed_weights(),
                                            self._pe_weights(ratio), self.mlp_mode, want_feat=True)
            self.rendcond = feat
            return sdf
        if not input.is_cuda:
            raise RuntimeError("recmv_b200.ImplicitNetwork runs on CUDA tensors only (no CPU path)")
        mode = ops.DEFAULT_MLP_MODE if self.mlp_mode is None else self.mlp_mode
        if self._fusable and self.train_fused and mode != ops.MLP_FP32_SIMT and input.dim() == 2:
            # training path: tensor-core layer GEMMs forward (outputs kept for the backward) + tensor-core backward
            # (ops.SdfMlpTrainFunction); weight-norm's W = g v / |v| stays a (tiny) torch graph so (g, v) receive
            # their gradients from dW
            self.last_path = "fused-train"
            Ws, bs = self.effective_weights()
            sdf, feat = ops.SdfMlpTrainFunction.apply(input.contiguous().float(), self._pe_weights(ratio), mode,
                                                      None,
                                                      *Ws, *bs)
            self.rendcond = feat
            return sdf
        self.last_path = "autograd-composite"
        return self._forward_graph(input, ratio)

    def _forward_graph(self, input, ratio):
        if self.embed_fn is not None:
            input = self.embed_fn(input, self._pe_weights(ratio))
        x = input
        for l in range(0, self.num_layers - 1):
            lin = getattr(self, "lin" + str(l))
            if l in self.skip_in:
                x = torch.cat([x, input], 1) / np.sqrt(2)
            x = lin(x)
            if l < self.num_layers - 2:
                x = self.softplus(x)
        if x.shape[-1] > self.d_out:
            self.rendcond = x[:, self.d_out:]
            x = x[:, 0:self.d_out]
        else:
            self.rendcond = None
        return x

    def value_and_grad(self, x, ratio, want_feat=False):
        """Fused (sdf, d sdf/d x) without an autograd graph: what the Newton step of the surface solve and
        inference-time normals need (utils/FindSurfacePs.py:176, OptimGarmentNetwork.py:3192).  One
        forward-mode launch; `rendcond` is updated when want_feat."""
        if not (self._fusable and x.is_cuda) or self.mlp_mode == ops.MLP_FP32_SIMT:
            xg = x.detach().clone().requires_grad_(True)
            with torch.enable_grad():
                y = self._forward_graph(xg, ratio)
                g = torch.autograd.grad(y.sum(), xg)[0]
            self.last_path = "autograd-composite"
            return y.detach(), g
        self.last_path = "fused-jvp"
        sdf, grad, feat = ops.sdf_value_and_grad(x.reshape(-1, 3), self.packed_weights(), self._pe_weights(ratio),
                                                 self.mlp_mode, want_feat)
        if want_feat:
            self.rendcond = feat
        return sdf, grad

    def gradient(self, x, y=None):
        x.requires_grad_(True)
        if y is None:
            y = self.forward(x, None)
        d_output = torch.ones_like(y, requires_grad=False, device=y.device)
        with ops.input_grad_only():   # second order on the tensor-core GEMMs (recmv_b200/second_order.py)
            gradients = torch.autograd.grad(outputs=y, inputs=x, grad_outputs=d_output, create_graph=True,
                                            retain_graph=True, only_inputs=True)[0]
        return gradients.view(-1, 3)


def getTmpSdf(device, multires, bias=0.6, feature_vector_size=256):
    """model/network.py:135-141."""
    net = ImplicitNetwork(feature_vector_size=feature_vector_size, d_in=3, d_out=1,
                          dims=[512, 512, 512, 512, 512, 512, 512, 512], geometric_init=True, bias=bias,
                          skip_in=[4], weight_norm=True, multires=multires)
    return net.to(device)
