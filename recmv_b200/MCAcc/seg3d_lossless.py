"""Coarse-to-fine ("lossless") evaluation of a query function on a voxel pyramid -- the sweep that feeds
marching cubes.  Same constructor, attributes (`spacing_{x,y,z}`, `b{x,y,z}`, `balance_value`,
`query_func`) and result as the reference's Seg3dLossless._forward (MCAcc/seg3d_lossless.py:233-428,
batch_eval :89-108), re-implemented with dense boolean masks instead of coordinate lists:

  * "already evaluated" is a bool lattice per level (the reference keeps `coords_accum` coordinate lists
    and re-sorts them with `unique(dim=1)` after every step, :367-370, :419-423);
  * the conflict loop works on a mask of the final lattice (reference: coordinate arithmetic + `unique`).

The set of voxels that get re-queried at every level is identical, so with the same `query_func` the
returned grid is bit-identical (tests/test_c2f_cpu.py compares against the imported reference class).
Every query goes through ONE fused launch of the SDF kernel when `query_func` is a recmv_b200
ImplicitNetwork under no_grad.
"""
import torch
import torch.nn as nn
import torch.nn.functional as F


def create_grid3D(min, max, steps, device="cuda:0"):
    """Lattice coordinates [N,3] (x,y,z), x fastest -- MCAcc/utils.py:88-101."""
    if type(min) is int:
        min = (min, min, min)
    if type(max) is int:
        max = (max, max, max)
    if type(steps) is int:
        steps = (steps, steps, steps)
    ax = [torch.linspace(float(min[i]), float(max[i]), int(steps[i])).long().to(device) for i in range(3)]
    gz, gy, gx = torch.meshgrid([ax[2], ax[1], ax[0]], indexing="ij")
    return torch.stack([gx, gy, gz]).view(3, -1).t()


class Seg3dLossless(nn.Module):
    def __init__(self, query_func, b_min, b_max, resolutions, channels=1, balance_value=0.5,
                 align_corners=False, visualize=False, debug=False, use_cuda_impl=False, faster=False,
                 use_shadow=False, **kwargs):
        super().__init__()
        self.query_func = query_func
        self.register_buffer('b_min', torch.as_tensor(b_min).float().view(1, 1, 3))
        self.register_buffer('b_max', torch.as_tensor(b_max).float().view(1, 1, 3))
        if type(resolutions[0]) is int:
            resolutions = torch.tensor([(r, r, r) for r in resolutions])
        else:
            resolutions = torch.tensor(resolutions)
        self.register_buffer('resolutions', resolutions)
        tmp = (self.b_max.view(3) - self.b_min.view(3)) / self.resolutions[-1].view(3).float()
        self.spacing_x, self.spacing_y, self.spacing_z = (tmp[i].item() for i in range(3))
        self.bx = self.b_min.view(-1)[0].item() + self.spacing_x / 2.
        self.by = self.b_min.view(-1)[1].item() + self.spacing_y / 2.
        self.bz = self.b_min.view(-1)[2].item() + self.spacing_z / 2.
        self.batchsize = 1
        self.balance_value = balance_value
        self.channels = channels
        assert channels == 1 and align_corners == False and visualize == False
        assert not faster and not use_shadow, "the _forward path of the reference is mirrored (faster / shadow are not)"
        # use_cuda_impl=True: the reference's optional fused upsampler (its own rounding, seg3d_lossless.py:267-268).
        # Default: the F.interpolate rounding -- evaluated by the same fused kernel on CUDA tensors (bit-identical to
        # the two torch interpolations + compare, see csrc/c2f.cu), by torch ops on CPU tensors.
        self.use_cuda_impl = use_cuda_impl
        self.align_corners = align_corners
        for r in resolutions:
            assert r[0] % 2 == 1 and r[1] % 2 == 1, f"resolution {r} need to be odd becuase of align_corner."
        self.register_buffer('smooth_w', torch.ones(1, 1, 3, 3, 3) / 27.0)
        self.stats = []

    # ---- query --------------------------------------------------------------------------------------
    def batch_eval(self, coords, **kwargs):
        """coords [1,M,3] integer lattice coordinates of the FINAL resolution -> [1,1,M]."""
        return self._eval(self.query_func, coords, **kwargs)

    def _eval(self, query_func, coords, **kwargs):
        """batch_eval with a given query function."""
        res = self.resolutions[-1].to(coords.device)
        step = 1.0 / res.float()
        c = coords.detach().float() / res + step / 2
        c = c * (self.b_max - self.b_min) + self.b_min
        occ = query_func(**kwargs, points=c)
        if type(occ) is list:
            occ = torch.stack(occ)
        assert occ.dim() == 3, "query_func should return a occupancy with shape of [bz, C, N]"
        return occ

    def _query_mask(self, mask, stride, occ, contiguous, **kwargs):
        """Evaluate the level-lattice voxels selected by `mask` [D,H,W]; returns (flat indices, interpolated
        values, queried values) and scatters the queried values into `occ` in place."""
        D, H, W = mask.shape
        # (x, y, z)-lexicographic order, z fastest: the order the reference issues its queries in
        # (`is_boundary.permute(2,1,0).nonzero()`, seg3d_lossless.py:311, and `unique(dim=0)`, :387) -- a
        # query function may round position-dependently inside a batch, so the order is part of parity
        xyz = mask.permute(2, 1, 0).nonzero(as_tuple=False)
        if xyz.shape[0] == 0:
            return xyz.new_zeros((0,)), None, None
        x, y, z = xyz[:, 0], xyz[:, 1], xyz[:, 2]
        idx = (z * H + y) * W + x
        # memory layout of the points as the reference hands them to query_func: the per-level sweep passes
        # nonzero()'s column-major [M,3] (strides (1,M)), the conflict loop a contiguous unique(dim=0) result
        coords = xyz * stride.view(1, 3)
        if contiguous:
            coords = coords.contiguous()
        flat = occ.view(-1)
        interp = flat[idx].clone()
        vals = self.batch_eval(coords.unsqueeze(0), **kwargs).view(-1).to(flat.dtype)
        flat[idx] = vals
        return idx, interp, vals

    # ---- device-worklist sweep ------------------------------------------------------------------------------------
    def _device_net(self):
        """(sdf_net, ratio) when `query_func` declares itself as a recmv_b200 ImplicitNetwork evaluated under no_grad
        (attribute `recmv_sdf`, set by recmv_b200.discretize / INTEGRATION.md) and the tensor-core engine can run it."""
        tag = getattr(self.query_func, "recmv_sdf", None)
        if tag is None or not self.b_min.is_cuda:
            return None
        net, ratio = tag
        from .. import ops
        mode = ops.DEFAULT_MLP_MODE if net.mlp_mode is None else net.mlp_mode
        if not getattr(net, "_fusable", False) or mode == ops.MLP_FP32_SIMT:
            return None
        return net, ratio, mode

    def _host_consts(self):
        """Host copies of the constant buffers the sweep's control flow needs (resolutions, box) and the coarse level's
        lattice coordinates (the reference registers those as its `init_coords` buffer): read back once per buffer version,
        not once per call -- the buffers live on the device, and every `int(v)` / `tolist()` on them is a blocking copy
        (25 of them per extraction before this cache)."""
        bufs = (self.resolutions, self.b_min, self.b_max)
        key = tuple((b.data_ptr(), b._version, str(b.device)) for b in bufs)
        hc = getattr(self, "_hc", None)
        if hc is None or hc[0] != key:
            res = [tuple(int(v) for v in r) for r in self.resolutions.cpu().tolist()]
            b_min, b_max = self.b_min.view(-1).cpu().tolist(), self.b_max.view(-1).cpu().tolist()
            dev = self.b_min.device
            final = torch.tensor(res[-1])
            coords = create_grid3D(0, final - 1, steps=torch.tensor(res[0]), device=dev).contiguous()
            hc = (key, res, b_min, b_max, coords)
            self._hc = hc
        return hc[1:]

    def _forward_device(self, net, ratio, mode):
        """Same sweep, same voxels re-queried, same arithmetic for the query points -- as a device worklist: per level
        ONE host read (statistics / overflow / "were there conflicts left"), no nonzero / unique / index scatter.
        The grid equals the torch-op path's bit for bit (tests/test_gpu_surface.py).  None on a worklist overflow."""
        sweep = _DeviceSweep(self, self.query_func, net, ratio, mode)
        self.stats = sweep.stats
        _run_sweeps([sweep])
        if sweep.failed:
            return None                                                      # worklist overflow: caller falls back
        self.last_sweep_path = "device-worklist"
        return sweep.occ

    def forward(self, **kwargs):
        devnet = self._device_net() if not kwargs else None
        if devnet is not None and not torch.is_grad_enabled():
            out = self._forward_device(*devnet)
            if out is not None:
                return out
        return self._forward_torch(**kwargs)

    def forward_many(self, query_funcs):
        """forward() for several query functions on this pyramid: one grid per function, each bit-identical to forward()
        with that function.  The device-worklist sweeps of all of them advance level by level together, so a level
        costs one host read for every network, not one per network (plus one per extra trip round the conflict loop
        that any of them needs).  A function that cannot use the worklist (no `recmv_sdf` tag, SIMT mode, not fusable,
        grad enabled) or whose worklist overflows takes forward()'s one-network fallback, _forward_torch.  Afterwards
        `query_func`, `stats` and `last_sweep_path` are the last function's, as after forward() on each in turn."""
        sweeps = [None] * len(query_funcs)
        if not torch.is_grad_enabled():
            for i, q in enumerate(query_funcs):
                self.query_func = q
                devnet = self._device_net()
                if devnet is not None:
                    sweeps[i] = _DeviceSweep(self, q, *devnet)
        _run_sweeps([s for s in sweeps if s is not None])
        out = []
        for q, s in zip(query_funcs, sweeps):
            self.query_func = q
            if s is not None and not s.failed:
                self.stats, self.last_sweep_path = s.stats, "device-worklist"
                out.append(s.occ)
            else:
                out.append(self._forward_torch())
        return out

    def _forward_torch(self, **kwargs):
        dev = self.b_min.device
        final = self.resolutions[-1].to(dev)
        Wf, Hf, Df = (int(v) for v in final)
        calculated = torch.zeros((Df, Hf, Wf), dtype=torch.bool, device=dev)
        occ, done = None, None
        self.stats = []
        for li, res in enumerate(self.resolutions):
            res = res.to(dev)
            W, H, D = (int(v) for v in res)
            stride = (final - 1) // (res - 1)
            sx, sy, sz = (int(v) for v in stride)
            if li == 0:
                # contiguous [N,3] like the reference's registered `init_coords` buffer (the memory layout of
                # the points reaches the query function and can change its rounding)
                coords = create_grid3D(0, final - 1, steps=res, device=dev).contiguous()
                occ = self.batch_eval(coords.unsqueeze(0), **kwargs).view(1, 1, D, H, W).float()
                done = torch.ones((D, H, W), dtype=torch.bool, device=dev)
                calculated[::sz, ::sy, ::sx] = True
                self.stats.append((W, H, D, D * H * W))
                continue
            fused = occ.is_cuda and not (torch.is_grad_enabled() and occ.requires_grad)
            if fused:
                from .. import ops
                occ, boundary = ops.interp2x_boundary3d_forward(occ.float().contiguous(), self.balance_value,
                                                                0 if self.use_cuda_impl else 1)
                self.last_sweep_path = "fused"
            elif self.use_cuda_impl:
                from .interp2x_boundary3d import Interp2xBoundary3dFunction
                occ, boundary = Interp2xBoundary3dFunction.apply(occ.float().contiguous(), self.balance_value)
                self.last_sweep_path = "fused-autograd"
            else:
                with torch.no_grad():
                    valid = F.interpolate((occ > self.balance_value).float(), size=(D, H, W), mode="trilinear",
                                          align_corners=True)
                occ = F.interpolate(occ.float(), size=(D, H, W), mode="trilinear", align_corners=True)
                boundary = (valid > 0.0) & (valid < 1.0)
                self.last_sweep_path = "torch"
            with torch.no_grad():
                done_up = torch.zeros((D, H, W), dtype=torch.bool, device=dev)
                done_up[::2, ::2, ::2] = done
                done = done_up
                if occ.is_cuda:
                    from .. import ops
                    todo = ops.c2f_todo_mask(boundary[0, 0].contiguous(), done)
                else:
                    boundary = (F.conv3d(boundary.float(), self.smooth_w, padding=1) > 0)[0, 0]
                    todo = boundary & ~done
            occ = occ.contiguous()
            queried = 0
            idx, interp, vals = self._query_mask(todo, stride, occ[0, 0], False, **kwargs)
            while idx.numel() > 0:
                queried += idx.numel()
                with torch.no_grad():
                    done.view(-1)[idx] = True
                    z, y, x = idx // (H * W), (idx // W) % H, idx % W
                    calculated[z * sz, y * sy, x * sx] = True
                    conflict = (interp - self.balance_value) * (vals - self.balance_value) < 0
                    if not bool(conflict.any()):
                        break
                    # 3x3x3 neighbourhood (in level-lattice steps) of every conflicting voxel, clamped to the
                    # lattice, minus everything already evaluated at ANY level
                    cmask = torch.zeros((D, H, W), dtype=torch.bool, device=dev)
                    cmask.view(-1)[idx[conflict]] = True
                    cmask = F.max_pool3d(cmask[None, None].float(), 3, stride=1, padding=1)[0, 0] > 0
                    cmask &= ~calculated[::sz, ::sy, ::sx]
                idx, interp, vals = self._query_mask(cmask, stride, occ[0, 0], True, **kwargs)
            self.stats.append((W, H, D, queried))
        return occ


class _DeviceSweep:
    """One network's device-worklist sweep, advanced one pyramid level at a time by _run_sweeps.  The constructor
    evaluates the coarse level; per finer level, begin() queues the refine pass and the first evaluation, rounds() queues
    two conflict rounds, and after_read() takes the level's counters once the driver has read them."""
    MORE, DONE, OVERFLOW = range(3)

    def __init__(self, engine, query_func, net, ratio, mode):
        self.dev = engine.b_min.device
        self.res, self.b_min, self.b_max, coords0 = engine._host_consts()
        self.balance, self.order = engine.balance_value, 0 if engine.use_cuda_impl else 1
        self.packed, self.pe_w, self.mode = net.packed_weights(), net._pe_weights(ratio), mode
        Wf, Hf, Df = self.res[-1]
        W, H, D = self.res[0]
        self.calculated = torch.zeros((Df, Hf, Wf), dtype=torch.uint8, device=self.dev)
        with torch.no_grad():
            self.occ = engine._eval(query_func, coords0.unsqueeze(0)).view(1, 1, D, H, W).float().contiguous()
        self.done = torch.ones((D, H, W), dtype=torch.uint8, device=self.dev)
        sx, sy, sz = self._stride(0)
        self.calculated[::sz, ::sy, ::sx] = 1
        self.stats = [(W, H, D, D * H * W)]
        self.lvl, self.li, self.failed = None, 0, False

    def _stride(self, li):
        (Wf, Hf, Df), (W, H, D) = self.res[-1], self.res[li]
        return (Wf - 1) // max(W - 1, 1), (Hf - 1) // max(H - 1, 1), (Df - 1) // max(D - 1, 1)

    def begin(self, li):
        from .. import ops
        W, H, D = self.res[li]
        total = D * H * W
        Dc, Hc, Wc = self.occ.shape[2:]
        self.li = li
        self.lvl = ops.C2fLevel((Dc, Hc, Wc), self.res[-1], self.b_min, self.b_max, self.dev,
                                total if total <= (1 << 22) else total // 4)
        self.occ, self.done = self.lvl.refine(self.occ, self.done, self.balance, self.order)
        self._evaluate()

    def _evaluate(self):
        self.lvl.evaluate(self.packed, self.pe_w, self.mode, self.occ, self.done, self.calculated, self.balance)

    def rounds(self):
        for _ in range(2):      # conflict rounds, queued speculatively (an empty list costs three near-empty launches)
            self.lvl.next_from_conflicts(self.calculated)
            self._evaluate()

    def after_read(self, counts):
        queried, conflicts, overflow = counts
        if overflow:
            self.failed = True
            return self.OVERFLOW
        if conflicts:
            return self.MORE
        self.stats.append(tuple(self.res[self.li]) + (queried,))
        self.lvl = None
        return self.DONE


def _run_sweeps(sweeps):
    """Advance every sweep (all on one pyramid) through the finer levels together: per level, each sweep's refine pass
    and two conflict rounds are queued, then ONE host read (ops.read_c2f_levels) serves every sweep still on that level;
    the ones with conflicts left get two more rounds and another shared read.  A sweep whose worklist overflows stops
    with `failed` set."""
    from .. import ops
    live = list(sweeps)
    for li in range(1, len(live[0].res) if live else 0):
        for s in live:
            s.begin(li)
        pending = live
        while pending:
            for s in pending:
                s.rounds()
            counts = ops.read_c2f_levels([s.lvl for s in pending])   # the level's one host synchronisation
            pending = [s for s, c in zip(pending, counts) if s.after_read(c) == s.MORE]
        live = [s for s in live if not s.failed]
