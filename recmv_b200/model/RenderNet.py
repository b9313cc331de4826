"""IDR colour MLP with the reference's API (model/RenderNet.py:10-103): cat[p, PE4(v), n, feat] = 289
-> 512 x4 ReLU -> 3 -> tanh, weight-normed.  Evaluated once per RAY (not per sample).  Without an autograd
graph (and for the standard 'idr' 289-wide configuration) the whole network is ONE launch of the tensor-core engine
(recmv_rendernet_fwd: input row assembled in shared memory, 5 layers on tensor cores, tanh in the epilogue);
with a graph it runs as torch ops over cuBLAS (SURVEY 8a row A8, 1.9 MFLOP/ray = 0.7 % of the per-ray work)."""
import torch
import torch.nn as nn

from .. import ops
from .Embedder import get_embedder, ratio_to_weights
from .packed import cached_pack


class RenderingNetwork_view_norm(nn.Module):
    def __init__(self, feature_vector_size, mode, d_in, d_out, dims, weight_norm=True, multires_n=0,
                 multires_v=0):
        super().__init__()
        self.mode = mode
        dims = [d_in + feature_vector_size] + dims + [d_out]
        self.embedv_fn = None
        self.multires_v = multires_v
        if multires_v > 0:
            self.embedv_fn, input_ch = get_embedder(multires_v)
            dims[0] += (input_ch - 3)
        self.embedn_fn = None
        self.multires_n = multires_n
        if multires_n > 0:
            self.embedn_fn, input_ch = get_embedder(multires_n)
            dims[0] += (input_ch - 3)
        self.num_layers = len(dims)
        for l in range(0, self.num_layers - 1):
            lin = nn.Linear(dims[l], dims[l + 1])
            if weight_norm:
                lin = nn.utils.weight_norm(lin)
            setattr(self, "lin" + str(l), lin)
        self.relu = nn.ReLU()
        self.tanh = nn.Tanh()
        self.mlp_mode = None
        self.train_fused = True   # grad-enabled forwards go through ops.RenderNetTrainFunction (False: torch graph)
        self.last_path = None
        self.fusable = (mode == 'idr' and multires_v == 4 and multires_n == 0 and feature_vector_size == 256
                        and d_in == 9 and d_out == 3 and list(dims[1:-1]) == [512] * 4)

    def effective_weights(self):
        Ws, bs = [], []
        for l in range(self.num_layers - 1):
            lin = getattr(self, "lin" + str(l))
            if hasattr(lin, "weight_g"):
                v, g = lin.weight_v, lin.weight_g
                Ws.append(v * (g / v.norm(dim=1, keepdim=True)))
            else:
                Ws.append(lin.weight)
            bs.append(lin.bias)
        return Ws, bs

    def packed_weights(self):
        return cached_pack(self, lambda: ops.rendernet_pack_weights(*self.effective_weights()))

    def forward(self, points, normals, view_dirs, feature_vectors, ratio):
        ratio = ratio['renderRatio']
        tensors = [points, normals, view_dirs, feature_vectors] + list(self.parameters())
        needs_graph = torch.is_grad_enabled() and any(t.requires_grad for t in tensors)
        if (self.fusable and points.is_cuda and points.dim() == 2 and not needs_graph
                and self.mlp_mode != ops.MLP_FP32_SIMT):
            self.last_path = "fused"
            return ops.rendernet_forward(points, normals, view_dirs, feature_vectors, self.packed_weights(),
                                         ratio_to_weights(self.multires_v, ratio), self.mlp_mode)
        if (self.fusable and self.train_fused and points.is_cuda and points.dim() == 2
                and self.mlp_mode != ops.MLP_FP32_SIMT):
            # training path: tensor-core layer GEMMs forward + backward (ops.RenderNetTrainFunction); tanh and the
            # weight-norm re-parametrisation stay (tiny) torch graphs
            self.last_path = "fused-train"
            Ws, bs = self.effective_weights()
            pre = ops.RenderNetTrainFunction.apply(points.contiguous().float(), normals.contiguous().float(),
                                                   view_dirs.contiguous().float(), feature_vectors.contiguous().float(),
                                                   ratio_to_weights(self.multires_v, ratio), *Ws, *bs)
            return self.tanh(pre)
        self.last_path = "autograd-composite"
        if self.embedv_fn is not None:
            view_dirs = self.embedv_fn(view_dirs, ratio_to_weights(self.multires_v, ratio))
        if self.embedn_fn is not None:
            normals = self.embedn_fn(normals, ratio_to_weights(self.multires_n, ratio))
        if self.mode == 'idr':
            x = torch.cat([points, view_dirs, normals, feature_vectors], dim=-1)
        elif self.mode == 'no_view_dir':
            x = torch.cat([points, normals, feature_vectors], dim=-1)
        elif self.mode == 'no_normal':
            x = torch.cat([points, view_dirs, feature_vectors], dim=-1)
        for l in range(0, self.num_layers - 1):
            x = getattr(self, "lin" + str(l))(x)
            if l < self.num_layers - 2:
                x = self.relu(x)
        return self.tanh(x)


def getRenderNet(device, conf):
    return RenderingNetwork_view_norm(conf.get_int('condlen'), d_in=9, d_out=3, dims=[512, 512, 512, 512],
                                      mode='idr', weight_norm=True, multires_v=conf.get_int('multires_v'),
                                      multires_n=conf.get_int('multires_n')).to(device)
