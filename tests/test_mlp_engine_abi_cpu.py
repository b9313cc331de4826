"""The fused MLP engine's C entry points, pinned without a device: the packed-blob sizes, and the status every entry
returns for argument errors it detects before any CUDA call (negative and zero sizes, each NULL pointer, an unknown
precision mode, a misaligned blob).  Several cases break more than one rule at once, so a change to the order of the
checks fails here as well as a change to a status code.

Device pointers are fake non-NULL addresses: every case returns before anything reads them.  The arguments the host
itself reads (the PE weights, the ray-march and voxel structs, the camera position) are real host arrays."""
import ctypes

import pytest

from recmv_b200 import _lib

OK, E_NULL, E_DTYPE, E_SHAPE, E_RANGE, E_UNSUPPORTED = 0, -1, -2, -3, -4, -5
TC3 = _lib.MLP_TC_F16X3
DEV = ctypes.c_void_p(1 << 20)                  # a fake, 1 KiB-aligned device address
MISALIGNED = ctypes.c_void_p((1 << 20) + 16)    # non-NULL, not 1 KiB-aligned


def _pe_w():
    return (ctypes.c_float * 12)(*([1.0] * 12))


def _vox(ws=DEV, D=4, H=4, W=4):
    return _lib.Voxel(ws_cl=ws, D=D, H=H, W=W, center=(ctypes.c_float * 3)(0, 0, 0), extend=1.0)


def _rm(samples=8):
    return _lib.RayMarch(cam_pos=(ctypes.c_float * 3)(0, 0, 3), t_near=1.0, t_far=5.0, samples_per_ray=samples)


# entry -> (argument names in C order, default arguments: a valid-looking call on fake device pointers, the pointers
# that must not be NULL)
ENTRIES = {
    "recmv_sdf_mlp_fwd": (
        "x packed pe_w out_sdf out_feat P mode stream",
        dict(x=DEV, packed=DEV, pe_w=_pe_w, out_sdf=DEV, out_feat=None, P=100, mode=TC3, stream=None),
        "x packed pe_w out_sdf"),
    "recmv_sdf_mlp_fwd_counted": (
        "x packed pe_w out_sdf out_feat capacity count_dev mode stream",
        dict(x=DEV, packed=DEV, pe_w=_pe_w, out_sdf=DEV, out_feat=None, capacity=100, count_dev=DEV, mode=TC3,
             stream=None),
        "x packed pe_w out_sdf count_dev"),
    "recmv_sdf_mlp_fwd_grad": (
        "x packed pe_w out_sdf out_feat out_grad P mode stream",
        dict(x=DEV, packed=DEV, pe_w=_pe_w, out_sdf=DEV, out_feat=None, out_grad=DEV, P=100, mode=TC3, stream=None),
        "x packed pe_w out_sdf out_grad"),
    "recmv_render_sdf": (
        "ray_dirs rm A trans frame_of_ray rays_per_frame num_frames vox packed pe_w out_sdf out_xc hit_idx hit_t R "
        "mode stream",
        dict(ray_dirs=DEV, rm=_rm, A=DEV, trans=DEV, frame_of_ray=None, rays_per_frame=10, num_frames=2, vox=_vox,
             packed=DEV, pe_w=_pe_w, out_sdf=DEV, out_xc=None, hit_idx=None, hit_t=None, R=20, mode=TC3,
             stream=None),
        "ray_dirs rm A trans vox packed pe_w out_sdf"),
    "recmv_deformer_fwd": (
        "ps conds batch_inds points_per_frame num_frames packed pe_w A trans vox out_translated out_offset "
        "out_posed P mode stream",
        dict(ps=DEV, conds=DEV, batch_inds=None, points_per_frame=50, num_frames=2, packed=DEV, pe_w=_pe_w, A=DEV,
             trans=DEV, vox=_vox, out_translated=DEV, out_offset=None, out_posed=DEV, P=100, mode=TC3, stream=None),
        "ps conds packed pe_w A trans vox"),
    "recmv_deformer_fwd_jac": (
        "ps conds batch_inds points_per_frame num_frames packed pe_w A trans vox out_translated out_offset "
        "out_posed out_jac P mode stream",
        dict(ps=DEV, conds=DEV, batch_inds=None, points_per_frame=50, num_frames=2, packed=DEV, pe_w=_pe_w, A=DEV,
             trans=DEV, vox=_vox, out_translated=None, out_offset=None, out_posed=DEV, out_jac=DEV, P=100, mode=TC3,
             stream=None),
        "ps conds packed pe_w A trans vox out_jac"),
    "recmv_rendernet_fwd": (
        "points normals view_dirs feats packed pe_w out_rgb P mode stream",
        dict(points=DEV, normals=DEV, view_dirs=DEV, feats=DEV, packed=DEV, pe_w=_pe_w, out_rgb=DEV, P=100, mode=TC3,
             stream=None),
        "points normals view_dirs feats packed pe_w out_rgb"),
    "recmv_surface_solve": (
        "cam_pos rays ps batch_inds sdf_packed sdf_pe_w tr_packed tr_pe_w conds num_frames A trans vox dthr athr "
        "w1 w2 times mode workspace workspace_bytes ok P stream",
        dict(cam_pos=lambda: (ctypes.c_float * 3)(0, 0, 3), rays=DEV, ps=DEV, batch_inds=None, sdf_packed=DEV,
             sdf_pe_w=_pe_w, tr_packed=DEV, tr_pe_w=_pe_w, conds=DEV, num_frames=2, A=DEV, trans=DEV, vox=_vox,
             dthr=1e-3, athr=1.0, w1=1.0, w2=1.0, times=3, mode=TC3, workspace=DEV, workspace_bytes=1 << 20, ok=DEV,
             P=100, stream=None),
        "cam_pos rays ps sdf_packed sdf_pe_w tr_packed tr_pe_w conds A trans vox workspace ok"),
}

# (entry, overrides, status)
CASES = []
for _name, (_args, _defaults, _required) in ENTRIES.items():
    _size = next(a for a in ("P", "capacity", "R") if a in _defaults)
    CASES += [(_name, {_size: -1}, E_SHAPE), (_name, {_size: -(1 << 40)}, E_SHAPE)]
    # a zero size returns before looking at any pointer but out_jac, which is checked first
    CASES.append((_name, {_size: 0, **{k: None for k, v in _defaults.items() if v is DEV and k != "out_jac"}}, OK))
    CASES += [(_name, {_k: None}, E_NULL) for _k in _required.split()]
    # an unknown mode; 0 (the fp32 SIMT kernel) only where tensor-core modes alone are accepted
    _mode_status = E_DTYPE if _name in ("recmv_sdf_mlp_fwd", "recmv_render_sdf") else E_UNSUPPORTED
    CASES += [(_name, {"mode": 7}, _mode_status), (_name, {"mode": -1}, _mode_status)]
    if _mode_status == E_UNSUPPORTED:
        CASES.append((_name, {"mode": _lib.MLP_FP32_SIMT}, E_UNSUPPORTED))

# NULL pointers the first NULL check does not cover, and the order of the checks
CASES += [
    # out_jac is checked before anything else
    ("recmv_deformer_fwd_jac", {"out_jac": None, "P": -1}, E_NULL),
    ("recmv_deformer_fwd_jac", {"out_jac": None, "P": 0}, E_NULL),
    ("recmv_deformer_fwd_jac", {"num_frames": 0}, E_SHAPE),
    ("recmv_deformer_fwd_jac", {"num_frames": 0, "P": 0}, E_SHAPE),
    ("recmv_deformer_fwd_jac", {"vox": lambda: _vox(ws=None)}, E_NULL),
    ("recmv_deformer_fwd_jac", {"ps": None, "mode": 7}, E_NULL),
    ("recmv_deformer_fwd_jac", {"out_posed": None, "A": None, "trans": None, "vox": None, "mode": 7}, E_UNSUPPORTED),
    ("recmv_deformer_fwd", {"num_frames": 0}, E_SHAPE),
    ("recmv_deformer_fwd", {"num_frames": -1, "P": 0}, E_SHAPE),
    ("recmv_deformer_fwd", {"vox": lambda: _vox(ws=None)}, E_NULL),
    ("recmv_deformer_fwd", {"out_posed": None, "A": None, "trans": None, "vox": None, "mode": 7}, E_UNSUPPORTED),
    ("recmv_deformer_fwd", {"P": -1, "ps": None}, E_SHAPE),
    ("recmv_rendernet_fwd", {"P": -1, "points": None, "mode": 7}, E_SHAPE),
    ("recmv_rendernet_fwd", {"points": None, "mode": 7}, E_NULL),
    ("recmv_sdf_mlp_fwd", {"P": -1, "x": None, "mode": 7}, E_SHAPE),
    ("recmv_sdf_mlp_fwd", {"x": None, "mode": 7}, E_NULL),
    ("recmv_sdf_mlp_fwd_counted", {"count_dev": None, "mode": 7}, E_NULL),
    ("recmv_sdf_mlp_fwd_grad", {"out_grad": None, "mode": 7}, E_NULL),
    ("recmv_render_sdf", {"vox": lambda: _vox(ws=None)}, E_NULL),
    ("recmv_render_sdf", {"rm": lambda: _rm(samples=0)}, E_SHAPE),
    ("recmv_render_sdf", {"rm": lambda: _rm(samples=-3)}, E_SHAPE),
    ("recmv_render_sdf", {"num_frames": 0}, E_SHAPE),
    ("recmv_render_sdf", {"vox": lambda: _vox(D=0)}, E_SHAPE),
    ("recmv_render_sdf", {"vox": lambda: _vox(H=-1)}, E_SHAPE),
    ("recmv_render_sdf", {"vox": lambda: _vox(W=0)}, E_SHAPE),
    ("recmv_render_sdf", {"num_frames": 0, "packed": None}, E_NULL),
    ("recmv_render_sdf", {"num_frames": 0, "mode": 7}, E_SHAPE),
    ("recmv_surface_solve", {"times": -1}, E_SHAPE),
    ("recmv_surface_solve", {"num_frames": 0}, E_SHAPE),
    ("recmv_surface_solve", {"num_frames": 0, "P": 0}, E_SHAPE),
    ("recmv_surface_solve", {"times": 0, "P": 0, "rays": None}, OK),
    ("recmv_surface_solve", {"workspace_bytes": 0}, E_SHAPE),
    ("recmv_surface_solve", {"workspace_bytes": 0, "ok": None}, E_NULL),
    ("recmv_surface_solve", {"workspace_bytes": 0, "mode": 7}, E_SHAPE),
]


def _call(name, overrides):
    lib = _lib.load()
    names, defaults, _ = ENTRIES[name]
    args = {**defaults, **overrides}
    vals = []
    for a in names.split():
        v = args[a]
        vals.append(v() if callable(v) else v)
    if name == "recmv_surface_solve" and "workspace_bytes" not in overrides:
        vals[names.split().index("workspace_bytes")] = max(lib.recmv_surface_solve_workspace(max(args["P"], 0)), 1)
    return getattr(lib, name)(*vals)


@pytest.mark.parametrize("name,overrides,status", CASES,
                         ids=[f"{n}-{'-'.join(f'{k}={getattr(v, '__name__', v)}' for k, v in o.items())}"
                              for n, o, _ in CASES])
def test_entry_argument_status(name, overrides, status):
    assert _call(name, overrides) == status


@pytest.mark.parametrize("net,nbytes", [("sdf", 16648192), ("translator", 4597760), ("rendernet", 4859904)])
def test_packed_bytes(net, nbytes):
    assert getattr(_lib.load(), f"recmv_{net}_packed_bytes")() == nbytes


@pytest.mark.parametrize("net", ["sdf", "translator", "rendernet"])
def test_pack_weights_argument_status(net):
    pack = getattr(_lib.load(), f"recmv_{net}_pack_weights")
    assert pack(None, DEV, DEV, None) == E_NULL
    assert pack(DEV, None, DEV, None) == E_NULL
    assert pack(DEV, DEV, None, None) == E_NULL
    assert pack(None, None, MISALIGNED, None) == E_NULL
    assert pack(DEV, DEV, MISALIGNED, None) == E_SHAPE
    assert pack(DEV, DEV, ctypes.c_void_p((1 << 20) + 512), None) == E_SHAPE


@pytest.mark.parametrize("mode", [7, -1, _lib.MLP_FP32_SIMT])
def test_set_acc_gain_rejects_unknown_modes(mode):
    assert _lib.load().recmv_tc_set_acc_gain(mode, 0.0) == E_DTYPE


@pytest.mark.parametrize("mode", [_lib.MLP_TC_F16X3, _lib.MLP_TC_F16X1])
@pytest.mark.parametrize("gain", [1e-4, -1.0, float("nan"), float("inf")])
def test_set_acc_gain_rejects_out_of_range_gains(mode, gain):
    assert _lib.load().recmv_tc_set_acc_gain(mode, gain) == E_RANGE
