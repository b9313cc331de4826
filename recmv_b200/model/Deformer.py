"""CompositeDeformer / MLPTranslator / LBSkinner with the reference's API (model/Deformer.py:22-34,
141-206, 216-531).  Buffer names of LBSkinner (b_min, b_max, ws, extra_trans, bbox_extend,
bbox_center, Js, init_pose) and parameter names of MLPTranslator (lin{0..4}.{weight,bias}) are kept so
reference checkpoints load.

LBSkinner.forward:
  * bone matrices A = G . init_pose are built on the host side in torch (24 joints, tiny);
  * no autograd needed -> ONE fused launch (voxel sample + blend + apply, recmv_lbs_fwd) over the
    channels-last cache of `ws` (rebuilt when `ws` changes, e.g. load_state_dict);
  * poses or translations that require grad (training) -> ops.LbsTrainFunction: the same forward kernel, and one
    backward kernel for the point / pose / translation gradients, on a chain built and differentiated by kernels
    (ops.BoneMatricesFunction);
  * otherwise with autograd (only the points, or train_fused = False, or a create_graph backward) -> the CUDA
    GridSamplerMine3dFunction (twice differentiable) + batched blend, without the reference's per-frame python loop and
    its `.item()` sync (Deformer.py:438-444).
"""
import numpy as np
import torch
import torch.nn as nn
import torch.nn.functional as F

from .. import ops
from .Embedder import get_embedder, ratio_to_weights


def quat2mat(quat):
    """utils/utils.py:21-38."""
    q = quat / quat.norm(p=2, dim=1, keepdim=True)
    w, x, y, z = q[:, 0], q[:, 1], q[:, 2], q[:, 3]
    B = quat.size(0)
    w2, x2, y2, z2 = w.pow(2), x.pow(2), y.pow(2), z.pow(2)
    wx, wy, wz = w * x, w * y, w * z
    xy, xz, yz = x * y, x * z, y * z
    return torch.stack([w2 + x2 - y2 - z2, 2 * xy - 2 * wz, 2 * wy + 2 * xz,
                        2 * wz + 2 * xy, w2 - x2 + y2 - z2, 2 * yz - 2 * wx,
                        2 * xz - 2 * wy, 2 * wx + 2 * yz, w2 - x2 - y2 + z2], dim=1).view(B, 3, 3)


def batch_rodrigues(theta):
    """smpl_pytorch.util.batch_rodrigues (un-vendored dependency of the reference; standard HMR
    form -- parity unpinned, see DESIGN.md)."""
    l1norm = torch.norm(theta + 1e-8, p=2, dim=1)
    angle = torch.unsqueeze(l1norm, -1)
    normalized = torch.div(theta, angle)
    angle = angle * 0.5
    quat = torch.cat([torch.cos(angle), torch.sin(angle) * normalized], dim=1)
    return quat2mat(quat)


class CompositeDeformer(nn.Module):
    def __init__(self, deformers):
        super().__init__()
        self.N = len(deformers)
        self.defs = nn.ModuleList(deformers)

    def forward(self, ps, conds, batch_inds=None, **kwargs):
        assert (self.N == len(conds))
        fused = self._fused_forward(ps, conds, batch_inds, kwargs)
        if fused is not None:
            return fused
        out = ps
        for cond, deformer in zip(conds, self.defs):
            out = deformer(out, cond, batch_inds, **kwargs)
        return out

    def value_and_jacobian(self, ps, conds, batch_inds, **kwargs):
        """(D(p) [P,3], J = dD/dp [P,3,3]) of [MLPTranslator, LBSkinner] in ONE forward-mode launch (no autograd
        graph; utils.compute_Jacobian semantics: row i = gradient of D_i).  None when this composite is not fusable."""
        return self._fused_forward(ps.detach(), conds, batch_inds, kwargs, want_jacobian=True)

    def device_solve_args(self, conds, ratio):
        """Everything `ops.surface_solve` needs from this deformer when it is the fusable [MLPTranslator, LBSkinner]
        composite on CUDA: (translator packed weights, translator PE weights, conds [F,128], skin tuple, mode);
        None otherwise."""
        if self.N != 2 or not isinstance(self.defs[0], MLPTranslator) or not isinstance(self.defs[1], LBSkinner):
            return None
        tr, sk = self.defs[0], self.defs[1]
        if not tr.fusable or tr.mlp_mode == ops.MLP_FP32_SIMT or not conds[0].is_cuda:
            return None
        poses, trans = conds[1]
        with torch.no_grad():
            A = sk.bone_matrices(poses)
            t = trans + sk.extra_trans
        center, extend = sk.bbox_host()
        return (tr.packed_weights(), ratio_to_weights(tr.multires, ratio['deformerRatio']), conds[0],
                (A, t, sk.ws_channels_last(), center, extend), tr.mlp_mode)

    def _fused_forward(self, ps, conds, batch_inds, kwargs, want_jacobian=False):
        """[MLPTranslator, LBSkinner] without an autograd graph -> ONE launch (translator MLP on the tensor cores, then
        the skinning-voxel sample + bone blend in the same kernel's epilogue)."""
        if self.N != 2 or not isinstance(self.defs[0], MLPTranslator) or not isinstance(self.defs[1], LBSkinner):
            return None
        tr, sk = self.defs[0], self.defs[1]
        if type(ps) == list or not ps.is_cuda or not tr.fusable or tr.mlp_mode == ops.MLP_FP32_SIMT:
            return None
        poses, trans = conds[1]
        tensors = [ps, conds[0], poses, trans] + list(tr.parameters())
        if not want_jacobian and torch.is_grad_enabled() and any(t.requires_grad for t in tensors):
            return None
        A = sk.bone_matrices(poses)
        center, extend = sk.bbox_host()
        ratio = kwargs['ratio']['deformerRatio']
        ppf = 0 if batch_inds is not None else ps.shape[1]
        res = ops.deformer_forward(ps.reshape(-1, 3), conds[0], tr.packed_weights(),
                                   ratio_to_weights(tr.multires, ratio), batch_inds, ppf,
                                   (A, trans + sk.extra_trans, sk.ws_channels_last(), center, extend),
                                   tr.mlp_mode, want_offset=True, want_translated=False, want_jacobian=want_jacobian)
        off, posed = res[1], res[2]
        tr.offset[kwargs.get('offset_type')] = off if batch_inds is not None else off.view(ps.shape[0], ps.shape[1], 3)
        tr.last_path = sk.last_path = "fused-deformer-jvp" if want_jacobian else "fused-deformer"
        posed = posed if batch_inds is not None else posed.view(ps.shape)
        return (posed, res[3]) if want_jacobian else posed


class MLPTranslator(nn.Module):
    """167 -> 512 x4 ReLU -> 3 offset MLP (model/Deformer.py:141-206)."""

    def __init__(self, feature_vector_size, multires, weight_norm=False):
        super().__init__()
        dims = [3 + feature_vector_size, 512, 512, 512, 512, 3]
        self.feature_vector_size = feature_vector_size
        self.embed_fn = None
        self.multires = multires
        if multires > 0:
            embed_fn, input_ch = get_embedder(multires)
            self.embed_fn = embed_fn
            dims[0] = input_ch + feature_vector_size
        self.num_layers = len(dims)
        for l in range(0, self.num_layers - 1):
            lin = nn.Linear(dims[l], dims[l + 1])
            if l == self.num_layers - 2:
                torch.nn.init.normal_(lin.weight, mean=0., std=0.001)
                torch.nn.init.constant_(lin.bias, 0.)
            setattr(self, "lin" + str(l), lin)
        self.relu = nn.ReLU()
        self.offset = {}
        self.mlp_mode = None
        self.train_fused = True   # grad-enabled forwards go through ops.TranslatorTrainFunction (False: torch graph)
        self.last_path = None
        self._packed, self._packed_key = None, None
        self.fusable = (multires == 6 and feature_vector_size == 128 and not weight_norm)

    def packed_weights(self):
        params = list(self.parameters())
        key = tuple((p.data_ptr(), p._version) for p in params)
        if self._packed is None or key != self._packed_key:
            with torch.no_grad():
                self._packed = ops.translator_pack_weights([getattr(self, "lin%d" % l).weight for l in range(5)],
                                                           [getattr(self, "lin%d" % l).bias for l in range(5)])
            self._packed_key = key
        return self._packed

    def forward(self, ps, conds, batch_inds=None, **kwargs):
        ratio = kwargs['ratio']['deformerRatio']
        offset_type = kwargs['offset_type']
        needs_graph = torch.is_grad_enabled() and (ps.requires_grad or conds.requires_grad
                                                   or any(p.requires_grad for p in self.parameters()))
        if self.fusable and ps.is_cuda and not needs_graph and self.mlp_mode != ops.MLP_FP32_SIMT:
            self.last_path = "fused"
            ppf = 0 if batch_inds is not None else ps.shape[1]
            tr, off, _ = ops.deformer_forward(ps.reshape(-1, 3), conds, self.packed_weights(),
                                              ratio_to_weights(self.multires, ratio), batch_inds, ppf, None,
                                              self.mlp_mode)
            if batch_inds is not None:
                self.offset[offset_type] = off
                return tr
            self.offset[offset_type] = off.view(ps.shape[0], ps.shape[1], 3)
            return tr.view(ps.shape[0], ps.shape[1], 3)
        if (self.fusable and self.train_fused and ps.is_cuda and self.mlp_mode != ops.MLP_FP32_SIMT
                and conds.dim() == 2):
            # training path: tensor-core layer GEMMs forward + backward (ops.TranslatorTrainFunction)
            self.last_path = "fused-train"
            flat = ps.reshape(-1, 3).contiguous().float()
            inds = batch_inds if batch_inds is not None else torch.arange(
                ps.shape[0], device=ps.device).repeat_interleave(ps.shape[1])
            off = ops.TranslatorTrainFunction.apply(flat, conds.contiguous().float(), inds.contiguous().long(),
                                                    ratio_to_weights(self.multires, ratio),
                                                    *[getattr(self, "lin%d" % l).weight for l in range(5)],
                                                    *[getattr(self, "lin%d" % l).bias for l in range(5)])
            if batch_inds is not None:
                self.offset[offset_type] = off
                return flat + off
            self.offset[offset_type] = off.view(ps.shape[0], ps.shape[1], 3)
            return ps + off.view(ps.shape[0], ps.shape[1], 3)
        self.last_path = "autograd-composite"
        if self.embed_fn is not None:
            ps = self.embed_fn(ps, ratio_to_weights(self.multires, ratio))
        if batch_inds is not None:
            x = torch.cat([ps, conds[batch_inds]], dim=1)
        else:
            x = torch.cat([ps, conds.view(-1, 1, self.feature_vector_size).expand(
                -1, ps.shape[1], self.feature_vector_size)], dim=-1).view(-1, ps.shape[-1] + self.feature_vector_size)
        for l in range(0, self.num_layers - 1):
            x = getattr(self, "lin" + str(l))(x)
            if l < self.num_layers - 2:
                x = self.relu(x)
        if batch_inds is not None:
            self.offset[offset_type] = x
            return ps[..., :3] + x
        self.offset[offset_type] = x.view(ps.shape[0], ps.shape[1], 3)
        return ps[..., :3] + x.view(ps.shape[0], ps.shape[1], 3)


def getTranslatorNet(device, conf):
    return MLPTranslator(conf.get_int('condlen'), multires=conf.get_int('multires')).to(device)


class LBSkinner(nn.Module):
    def __init__(self, ws, bmins, bmaxs, Js, parents, init_pose=None, align_corners=False,
                 extra_trans=None, bbox_extend=None, bbox_center=None):
        super().__init__()

        def as_buf(v):
            if type(v) is list:
                return torch.tensor(v, dtype=torch.float).view(1, 3)
            if type(v) is np.ndarray:
                return torch.from_numpy(v.astype(np.float32)).view(1, 3)
            return v.view(1, 3)
        self.register_buffer('b_min', as_buf(bmins))
        self.register_buffer('b_max', as_buf(bmaxs))
        if type(ws) is np.ndarray:
            ws = torch.from_numpy(ws.astype(np.float32))
        self.register_buffer('ws', ws.to(torch.float))
        if extra_trans is None:
            extra_trans = torch.full([1, 3], 0.).float()
        self.register_buffer('extra_trans', extra_trans.to(torch.float))
        self.register_buffer('bbox_extend', torch.as_tensor(bbox_extend).to(torch.float))
        self.register_buffer('bbox_center', torch.as_tensor(bbox_center).to(torch.float))
        self.align_corners = align_corners
        assert (align_corners == False)
        self.register_buffer('Js', Js.view(24, 3))
        self.parents = parents
        if init_pose is None:
            self.register_buffer('init_pose', None)
        else:
            if type(init_pose) == np.ndarray:
                init_pose = torch.from_numpy(init_pose.astype(np.float32))
            if init_pose.numel() == 24 * 3:
                self.init_pose_inverse(batch_rodrigues(init_pose.view(-1, 3)).view(24, 3, 3), self.Js)
            else:
                self.register_buffer('init_pose', init_pose.view(24, 4, 4))
        self._ws_cl = None
        self._ws_key = None
        self._bbox_key, self._bbox_host = None, None
        self._parents_i32 = None
        self.train_fused = True   # poses / trans that require grad: kernel chain + ops.LbsTrainFunction (False: torch graph)
        self.last_path = None

    @property
    def last_backward(self):
        """Which backward branch of ops.LbsTrainFunction ran last: "fused" or "autograd-composite (create_graph)"."""
        return ops.LbsTrainFunction.last_backward

    def bbox_size(self):
        margin = torch.tensor([0.15, 0.15, 0.20]).to(self.b_min)
        return self.b_min - margin, self.b_max + margin

    def init_pose_inverse(self, init_pose, Js):
        """model/Deformer.py:280-303."""
        resultsR = [init_pose[0]]
        resultsT = [Js[0]]
        for i in range(1, self.parents.shape[0]):
            j_here = Js[i] - Js[self.parents[i]]
            resultsR.append(resultsR[self.parents[i]].matmul(init_pose[i]))
            resultsT.append(resultsR[self.parents[i]].matmul(j_here.view(-1, 1)).view(-1) + resultsT[self.parents[i]])
        invs = []
        for R, T in zip(resultsR, resultsT):
            inv = torch.zeros(4, 4)
            inv[3, 3] = 1.
            inv[:3, :3] = R.transpose(0, 1)
            inv[:3, 3] = (-T.view(1, -1).matmul(R)).view(-1)
            invs.append(inv)
        self.register_buffer('init_pose', torch.stack(invs, dim=0))

    # -- skeleton ---------------------------------------------------------------------------------
    def _chain(self, poses):
        batch_size = poses.shape[0]
        R = batch_rodrigues(poses.view(-1, 3)).view(batch_size, 24, 3, 3)
        Js = self.Js.view(1, 24, 3, 1).expand(batch_size, 24, 3, 1)

        def make_A(Rm, t):
            R_homo = F.pad(Rm, [0, 0, 0, 1, 0, 0])
            t_homo = torch.cat([t, torch.ones(Rm.shape[0], 1, 1).to(Rm.device)], dim=1)
            return torch.cat([R_homo, t_homo], 2)
        results = [make_A(R[:, 0], Js[:, 0])]
        parent = self.parents
        for i in range(1, parent.shape[0]):
            results.append(torch.matmul(results[int(parent[i])], make_A(R[:, i], Js[:, i] - Js[:, int(parent[i])])))
        return torch.stack(results, dim=1), Js

    def bbox_host(self):
        """(center [3] floats, extend float) of the voxel normalisation as HOST values, cached against the buffers'
        (data_ptr, _version): the kernels take them by value, and reading CUDA buffers per call would cost two
        blocking D2H syncs on every deformer launch."""
        key = (self.bbox_center.data_ptr(), self.bbox_center._version, self.bbox_extend.data_ptr(), self.bbox_extend._version)
        if self._bbox_key != key:
            self._bbox_host = (self.bbox_center.view(-1)[:3].tolist(), float(self.bbox_extend.view(-1)[0]))
            self._bbox_key = key
        return self._bbox_host

    def _parents_dev(self, device):
        if self._parents_i32 is None or self._parents_i32.device != device:
            self._parents_i32 = torch.as_tensor(self.parents).to(torch.int32).to(device).contiguous()
        return self._parents_i32

    def _chain_graph(self, poses):
        """True when the poses need a graph and it is the device chain's (ops.BoneMatricesFunction)."""
        return poses.is_cuda and self.train_fused and torch.is_grad_enabled() and poses.requires_grad

    def bone_matrices(self, poses):
        """A [N,24,4,4] = G . init_pose (Deformer.py:372-405).  One kernel when no graph is needed; with a graph, the same
        kernel forward and its VJP kernel backward (train_fused), or the torch chain."""
        if poses.is_cuda and not (torch.is_grad_enabled() and poses.requires_grad):
            return ops.bone_matrices(poses.reshape(-1, 24, 3), self.Js, self._parents_dev(poses.device), self.init_pose)[1]
        if self._chain_graph(poses):
            return ops.BoneMatricesFunction.apply(poses.reshape(-1, 24, 3).float(), self.Js, self._parents_dev(poses.device),
                                                  self.init_pose)[1]
        results, Js = self._chain(poses)
        batch_size = poses.shape[0]
        if self.init_pose is None:
            Js_w0 = torch.cat([Js, torch.zeros(batch_size, 24, 1, 1).to(poses.device)], dim=2)
            init_bone = F.pad(torch.matmul(results, Js_w0), [3, 0, 0, 0, 0, 0, 0, 0])
            return results - init_bone
        return torch.matmul(results, self.init_pose.view(1, 24, 4, 4).expand(batch_size, 24, 4, 4))

    def posedSkeleton(self, conds):
        poses, trans = conds
        assert (poses.shape[0] == trans.shape[0])
        if poses.is_cuda and not (torch.is_grad_enabled() and poses.requires_grad):
            G, _ = ops.bone_matrices(poses.reshape(-1, 24, 3), self.Js, self._parents_dev(poses.device), None, want_A=False)
            return G[:, :, :3, 3]
        if self._chain_graph(poses):
            G, _ = ops.BoneMatricesFunction.apply(poses.reshape(-1, 24, 3).float(), self.Js, self._parents_dev(poses.device),
                                                  None)
            return G[:, :, :3, 3]
        results, _ = self._chain(poses)
        return results[:, :, :3, 3]

    def inv_transform_v(self, v, scale_grid, transl):
        v = v - transl[None, None]
        v = v / scale_grid
        v = v * 2
        return v

    def ws_channels_last(self):
        key = (self.ws.data_ptr(), self.ws._version)
        if self._ws_cl is None or key != self._ws_key:
            if self.ws.shape[1] != 24:
                raise RuntimeError("LBSkinner expects a 24-channel skinning voxel")
            self._ws_cl = ops.voxel_to_channels_last(self.ws.contiguous())
            self._ws_key = key
        return self._ws_cl

    # ColorBrewer "Paired" entries 1 / 3 / 5 (what matplotlib's get_cmap('Paired').colors holds) and white, per
    # joint: engineer/utils/skinning_weights.py:5-52
    _JOINT_COLORS = None

    def query_skinning_weights_colors(self, tps):
        """model/Deformer.py:331-340: per-point colour = skinning weights [P,24] x fixed joint colours; CPU float64
        tensor [P,3] like the reference (torch CPU weights times a float64 numpy table)."""
        if LBSkinner._JOINT_COLORS is None:
            blue, green, red, white = (31 / 255, 120 / 255, 180 / 255), (51 / 255, 160 / 255, 44 / 255), \
                (227 / 255, 26 / 255, 28 / 255), (1.0, 1.0, 1.0)
            names = "w b g r w w w g b r w w w b g r g b w w b g w w".split()   # cyan -> Paired[3], darkgreen -> Paired[1]
            LBSkinner._JOINT_COLORS = torch.tensor([{"w": white, "b": blue, "g": green, "r": red}[n] for n in names],
                                                   dtype=torch.float64)
        pts = tps.reshape(-1, 3)
        if pts.is_cuda:
            with torch.no_grad():
                center, extend = self.bbox_host()
                ident = torch.eye(4, device=pts.device).expand(1, 24, 4, 4).contiguous()
                _, w = ops.lbs_forward(pts, ident, torch.zeros((1, 3), device=pts.device), self.ws_channels_last(),
                                       center, extend, None, pts.shape[0], None, want_weights=True)
        else:
            raise RuntimeError("recmv_b200.LBSkinner runs on CUDA tensors only (no CPU path)")
        return (w.detach().cpu().double()[:, :, None] * LBSkinner._JOINT_COLORS[None]).sum(1)

    def repose(self, ps, conds, batch_inds=None, **kwargs):
        """model/Deformer.py:446-531: `forward` without the extra translation (used when re-posing canonical
        geometry for animation)."""
        return self._warp(ps, conds, batch_inds, add_extra=False)

    def forward(self, ps, conds, batch_inds=None, **kwargs):
        return self._warp(ps, conds, batch_inds, add_extra=True)

    def _warp(self, ps, conds, batch_inds, add_extra):
        if type(ps) == list:
            tps, ps = ps
        else:
            tps = ps
        poses, trans = conds
        if add_extra:
            trans = trans + self.extra_trans
        batch_size = poses.shape[0]
        assert (batch_size == trans.shape[0])
        A = self.bone_matrices(poses)
        needs_graph = torch.is_grad_enabled() and any(
            t.requires_grad for t in (ps, tps, poses, trans))
        if not ps.is_cuda:
            raise RuntimeError("recmv_b200.LBSkinner runs on CUDA tensors only (no CPU path)")
        center, extend = self.bbox_host()
        if not needs_graph:
            self.last_path = "fused"
            if batch_inds is None:
                bsz, pnum, _ = ps.shape
                assert (batch_size == bsz)
                out = ops.lbs_forward(ps.reshape(-1, 3), A, trans, self.ws_channels_last(), center, extend,
                                      None, pnum, None if tps is ps else tps.reshape(-1, 3))
                return out.view(bsz, pnum, 3)
            out = ops.lbs_forward(ps.reshape(-1, 3), A, trans, self.ws_channels_last(), center, extend,
                                  batch_inds, 0, None if tps is ps else tps.reshape(-1, 3))
            return out
        if self.train_fused and torch.is_grad_enabled() and (poses.requires_grad or trans.requires_grad):
            # training step: forward kernel, backward kernel for the pose / translation / point gradients
            self.last_path = "fused-train"
            p32 = ps.float().contiguous()
            t32 = None if tps is ps else tps.float().contiguous()
            bi = None if batch_inds is None else batch_inds.contiguous().long()
            if bi is None:
                assert (batch_size == ps.shape[0])
            return ops.LbsTrainFunction.apply(p32, t32, A.float(), trans.float().contiguous(), bi,
                                              (self.ws_channels_last(), center, extend),
                                              lambda p, t, a, tr: self._composite(p, p if t is None else t, a, tr, bi))
        self.last_path = "autograd-composite"
        return self._composite(ps, tps, A, trans, batch_inds)

    def _composite(self, ps, tps, A, trans, batch_inds):
        """The skinning as a torch graph on the CUDA sampler (twice differentiable)."""
        batch_size = A.shape[0]
        nps = self.inv_transform_v(tps, self.bbox_extend, self.bbox_center).view(-1, 3)
        # the frozen voxel in its cached channels-last layout (one corner = 24 contiguous floats = 3 sectors instead of the
        # reference layout's 24)
        ws_cl = self.ws_channels_last()
        ps_ws = ops.FrozenVoxelSampleFunction.apply(ws_cl.view(1, *ws_cl.shape), nps.reshape(1, 1, 1, -1, 3))
        ps_ws = ps_ws.view(-1, nps.shape[0]).transpose(0, 1)
        if batch_inds is None:
            bsz, pnum, _ = ps.shape
            T = torch.matmul(ps_ws.view(bsz, pnum, 24), A.view(batch_size, 24, 16)).view(bsz, pnum, 4, 4)
            vh = torch.cat([ps, torch.ones(bsz, pnum, 1, device=ps.device)], dim=2)
            return torch.matmul(T, vh.unsqueeze(-1))[:, :, :3, 0] + trans.view(-1, 1, 3)
        ps = ps.reshape(-1, 3)
        T = torch.einsum('pj,pjk->pk', ps_ws, A.view(batch_size, 24, 16)[batch_inds]).view(-1, 4, 4)
        vh = F.pad(ps, (0, 1), mode='constant', value=1).unsqueeze(-1)
        return torch.matmul(T, vh)[:, :3, 0] + trans[batch_inds]

    def inverse(self, x_obs, conds, batch_inds=None):
        """North-star inverse warp (observation -> canonical) with the FastMinv singularity rule."""
        poses, trans = conds
        trans = trans + self.extra_trans
        A = self.bone_matrices(poses)
        center, extend = self.bbox_host()
        shp = x_obs.shape
        ppf = 0 if batch_inds is not None else (x_obs.shape[1] if x_obs.dim() == 3 else x_obs.shape[0])
        xc, ok = ops.lbs_inverse(x_obs.reshape(-1, 3), A, trans, self.ws_channels_last(), center, extend,
                                 batch_inds, ppf)
        return xc.view(shp), ok


# -- skinning-voxel construction (model/Deformer.py:533-623): setup work, run once per body ----------------------------
def _host3(v):
    return [float(x) for x in torch.as_tensor(v).float().view(-1).tolist()]


def _lbsw_field(bmins, bmaxs, resolutions, smpl_verts, smpl_ws, align_corners, mean_neighbor, smooth_times, zero_below):
    """(ws [1,24,D,H,W], its channels-last copy [D,H,W,24]): the kNN blend kernel, then the smoothing kernel."""
    if not smpl_verts.is_cuda:
        raise RuntimeError("compute_lbswField runs on CUDA tensors only (no CPU path)")
    verts = smpl_verts.reshape(-1, 3).float().contiguous()
    vert_ws = smpl_ws.reshape(verts.shape[0], -1).float().contiguous()
    ws_cl = ops.lbsw_knn_blend(verts, vert_ws, _host3(bmins), _host3(bmaxs), resolutions, mean_neighbor, align_corners)
    return ops.lbsw_smooth(ws_cl, smooth_times, zero_below)


def smooth_weights(weights, times=3):
    """model/Deformer.py:533-544 on a [1,24,D,H,W] CUDA voxel (returns a new tensor; `weights` is left as it is)."""
    if not weights.is_cuda:
        raise RuntimeError("smooth_weights runs on CUDA tensors only (no CPU path)")
    return ops.lbsw_smooth(ops.voxel_to_channels_last(weights.float().contiguous()), times)[0]


def compute_lbswField(bmins, bmaxs, resolutions, smpl_verts, smpl_ws, align_corners=False, mean_neighbor=5,
                      smooth_times=30):
    """model/Deformer.py:546-591 -> ws [1,24,D,H,W] on the device of smpl_verts (CUDA only).  Two kernels instead of
    38 chunks of a [50000, V, 3] difference tensor; the k-th-distance ties that torch.topk leaves undefined go to the
    lower vertex index."""
    return _lbsw_field(bmins, bmaxs, resolutions, smpl_verts, smpl_ws, align_corners, mean_neighbor, smooth_times, 0.0)[0]


def skinner_from_body(verts, vert_ws, Js, parents, pose, resolution, extra_trans=None):
    """The part of initialLBSkinner after SMPL (model/Deformer.py:603-623), line by line: the field is built over the
    vertices' tight [min, max] box, the skinner normalises with its centre and 1.1 x its largest extent.
    verts [V,3] (or [1,V,3]), vert_ws [V,24], Js [24,3], parents [24], pose (24 x 3 axis-angle).
    Returns (LBSkinner, verts [V,3], None); the skinner's channels-last cache is already filled."""
    verts = verts.reshape(-1, 3)
    bbox_data_min = verts.min(0).values
    bbox_data_max = verts.max(0).values
    bbox_data_extend = (bbox_data_max - bbox_data_min).max()
    bbox_grid_extend = bbox_data_extend * 1.1
    grid_center = (bbox_data_min + bbox_data_max) / 2
    ws, ws_cl = _lbsw_field(bbox_data_min.tolist(), bbox_data_max, resolution, verts, vert_ws.reshape(verts.shape[0], 24),
                            False, 30, 30, 0.0)
    sk = LBSkinner(ws, bbox_data_min, bbox_data_max, Js, parents, init_pose=pose, align_corners=False,
                   extra_trans=extra_trans, bbox_extend=bbox_grid_extend, bbox_center=grid_center)
    sk._ws_cl, sk._ws_key = ws_cl, (sk.ws.data_ptr(), sk.ws._version)
    return sk, verts, None


def initialLBSkinner(gender, shape, pose, resolution, bmins=None, bmaxs=None, extra_trans=None):
    """model/Deformer.py:594-623.  SMPL itself is not part of this package: `smpl_pytorch` is imported here, as the
    reference does at module level."""
    from smpl_pytorch.SMPL import getSMPL
    smpl = getSMPL(gender).to(shape.device)
    Js, _ = smpl.skeleton(shape.view(1, -1), True)
    verts, _, _ = smpl(shape.view(1, -1), pose.view(1, 24, 3), True)
    if bmins is not None and bmaxs is not None:
        # the reference defines its box only in the adaptive branch, so given boxes fail at Deformer.py:612
        raise UnboundLocalError("local variable 'bbox_data_min' referenced before assignment")
    sk, v, _ = skinner_from_body(verts.view(6890, 3), smpl.weight.view(6890, 24), Js, smpl.parents, pose, resolution,
                                 extra_trans)
    return sk, v, torch.tensor(smpl.faces, dtype=torch.long, device=verts.device)
