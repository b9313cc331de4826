"""CPU: every public wrapper in ops.py that hands caller tensors to a kernel refuses a bad operand with a RuntimeError
that names the wrapper and the operand, before it allocates, sizes or launches anything.  One row per wrapper holds
valid-shaped operands on the CPU: the row itself is refused for not being on CUDA, and each operand with the wrong
dtype, any bound extent changed by one, or as a strided view is refused for that reason, never reaching _launch."""
import ast
import inspect
import re

import pytest
import torch

from recmv_b200 import ops


def f32(*s):
    return torch.zeros(s)


def i64(*s):
    return torch.zeros(s, dtype=torch.int64)


def i32(*s):
    return torch.zeros(s, dtype=torch.int32)


def bool_(*s):
    return torch.zeros(s, dtype=torch.bool)


def packed(net):
    return torch.zeros((ops._packed_bytes(net),), dtype=torch.uint8)


BOX = ((0.0, 0.0, 0.0), 1.0)      # voxel centre and extent
A, TRANS, WS_CL = f32(2, 24, 4, 4), f32(2, 3), f32(3, 4, 5, 24)


def row(fn, call, operands, free="", conv="", cont="", covers=None, shape_error=RuntimeError):
    """fn: the wrapper's name in its messages; call(o) runs it on the operands o {name: tensor}; free: "name:dim" extents
    no other operand binds; conv: operands the wrapper converts (dtype and layout) itself, cont: those it only makes
    contiguous; covers: the ops.py functions / Functions the row drives."""
    return dict(fn=fn, call=call, ops=operands, free=set(free.split()), conv=set(conv.split()),
                cont=set(cont.split()) | set(conv.split()), covers=set((covers or fn).split()), shape_error=shape_error)


def _lbs(o, fn, *names):
    return fn(*[o[n] for n in names[:3]], o["ws_cl"], *BOX, o["batch_inds"], 0, *[o[n] for n in names[3:]])


ROWS = [
    row("minv3x3", lambda o: ops.minv3x3(o["ms"]), dict(ms=f32(4, 3, 3)), "ms:0"),
    row("minv3x3_backward", lambda o: ops.minv3x3_backward(o["grads"], o["invs"]),
        dict(grads=f32(4, 3, 3), invs=f32(4, 3, 3))),
    row("grid_sample3d_forward", lambda o: ops.grid_sample3d_forward(o["input"], o["grid"]),
        dict(input=f32(2, 3, 4, 5, 6), grid=f32(2, 1, 2, 7, 3)), "input:1 input:2 input:3 input:4 grid:1 grid:2 grid:3"),
    row("grid_sample3d_backward", lambda o: ops.grid_sample3d_backward(o["input"], o["grid"], o["grad_output"]),
        dict(input=f32(2, 3, 4, 5, 6), grid=f32(2, 1, 2, 7, 3), grad_output=f32(2, 3, 1, 2, 7)),
        "input:2 input:3 input:4", cont="grad_output"),
    row("grid_sample3d_dbackward",
        lambda o: ops.grid_sample3d_dbackward(o["gg_input"], o["gg_grid"], o["input"], o["grid"], o["grad_output"]),
        dict(gg_input=f32(2, 3, 4, 5, 6), gg_grid=f32(2, 1, 2, 7, 3), input=f32(2, 3, 4, 5, 6), grid=f32(2, 1, 2, 7, 3),
             grad_output=f32(2, 3, 1, 2, 7)), cont="gg_input gg_grid grad_output"),
    row("voxel_to_channels_last", lambda o: ops.voxel_to_channels_last(o["ws"]), dict(ws=f32(1, 3, 4, 5, 6)),
        "ws:1 ws:2 ws:3 ws:4"),
    row("lbsw_knn_blend", lambda o: ops.lbsw_knn_blend(o["verts"], o["vert_ws"], (0, 0, 0), (1, 1, 1), (4, 4, 4), 2),
        dict(verts=f32(5, 3), vert_ws=f32(5, 24)), "vert_ws:1"),
    row("lbsw_smooth", lambda o: ops.lbsw_smooth(o["ws_cl"], 1), dict(ws_cl=WS_CL), "ws_cl:0 ws_cl:1 ws_cl:2"),
    row("mc_gpu_many", lambda o: ops.mc_gpu_many([o["grids[0]"]], [(1, 1, 1)], [(0, 0, 0)]),
        {"grids[0]": f32(4, 5, 6)}, "grids[0]:0 grids[0]:1 grids[0]:2"),
    row("vertex_faces", lambda o: ops.vertex_faces(o["faces"], 5), dict(faces=i64(4, 3)), "faces:0"),
    row("make_voxel", lambda o: ops.make_voxel(o["ws_cl"], *BOX), dict(ws_cl=WS_CL), "ws_cl:0 ws_cl:1 ws_cl:2"),
    row("lbs_forward", lambda o: _lbs(o, ops.lbs_forward, "ps", "A", "trans", "tps"),
        dict(ps=f32(6, 3), A=A, trans=TRANS, ws_cl=WS_CL, batch_inds=i64(6), tps=f32(6, 3)),
        "ws_cl:0 ws_cl:1 ws_cl:2", conv="ps A trans batch_inds tps"),
    row("lbs_inverse", lambda o: _lbs(o, ops.lbs_inverse, "x_obs", "A", "trans"),
        dict(x_obs=f32(6, 3), A=A, trans=TRANS, ws_cl=WS_CL, batch_inds=i64(6)),
        "ws_cl:0 ws_cl:1 ws_cl:2", conv="x_obs A trans batch_inds"),
    row("lbs_backward", lambda o: _lbs(o, ops.lbs_backward, "ps", "A", "grad_out", "tps"),
        dict(ps=f32(6, 3), A=A, grad_out=f32(6, 3), ws_cl=WS_CL, batch_inds=i64(6), tps=f32(6, 3)),
        "A:0 ws_cl:0 ws_cl:1 ws_cl:2", conv="ps A grad_out batch_inds tps"),
    row("lbs_vjp_backward", lambda o: _lbs(o, ops.lbs_vjp_backward, "ps", "A", "grad_out", "tps", "cot_ps", "cot_tps"),
        dict(ps=f32(6, 3), A=A, grad_out=f32(6, 3), ws_cl=WS_CL, batch_inds=i64(6), tps=f32(6, 3), cot_ps=f32(6, 3),
             cot_tps=f32(6, 3)), "A:0 ws_cl:0 ws_cl:1 ws_cl:2", conv="ps A grad_out batch_inds tps cot_ps cot_tps"),
    row("bone_matrices", lambda o: ops.bone_matrices(o["poses"], o["Js"], o["parents_i32"], o["init_pose"]),
        dict(poses=f32(2, 24, 3), Js=f32(24, 3), parents_i32=i32(24), init_pose=f32(24, 4, 4)), "poses:0",
        conv="poses Js init_pose"),
    row("bone_matrices_backward",
        lambda o: ops.bone_matrices_backward(o["poses"], o["Js"], o["parents_i32"], o["init_pose"], o["G"], o["dG"],
                                             o["dA"]),
        dict(poses=f32(2, 24, 3), Js=f32(24, 3), parents_i32=i32(24), init_pose=f32(24, 4, 4), G=A, dG=A, dA=A),
        conv="poses Js init_pose dG dA", cont="G"),
    row("translator_pack_weights",
        lambda o: ops.translator_pack_weights([f32(*s) for s in ops.TRANSLATOR_LAYER_SHAPES],
                                              [f32(s[0]) for s in ops.TRANSLATOR_LAYER_SHAPES]),
        {}, covers="_pack_weights"),
    row("sdf_mlp_forward", lambda o: ops.sdf_mlp_forward(o["x"], o["packed"]), dict(x=f32(6, 3), packed=packed("sdf")),
        "x:0", conv="x"),
    row("sdf_value_and_grad", lambda o: ops.sdf_value_and_grad(o["x"], o["packed"]),
        dict(x=f32(6, 3), packed=packed("sdf")), "x:0", conv="x"),
    row("deformer_forward",
        lambda o: ops.deformer_forward(o["ps"], o["conds"], o["packed"], None, o["batch_inds"], 0,
                                       (o["A"], o["trans"], o["ws_cl"], *BOX)),
        dict(ps=f32(6, 3), conds=f32(2, 128), packed=packed("translator"), batch_inds=i64(6), A=A, trans=TRANS,
             ws_cl=WS_CL), "ws_cl:0 ws_cl:1 ws_cl:2", conv="ps conds batch_inds A trans"),
    row("rendernet_forward",
        lambda o: ops.rendernet_forward(o["points"], o["normals"], o["view_dirs"], o["feature_vectors"], o["packed"],
                                        [1.0] * 8),
        dict(points=f32(6, 3), normals=f32(6, 3), view_dirs=f32(6, 3), feature_vectors=f32(6, 256),
             packed=packed("rendernet")), conv="points normals view_dirs feature_vectors"),
    row("render_sdf",
        lambda o: ops.render_sdf(o["ray_dirs"], (0, 0, 0), 0.1, 2.0, 8, o["A"], o["trans"], o["ws_cl"], *BOX,
                                 o["packed"], frame_of_ray=o["frame_of_ray"], out_sdf=o["out_sdf"]),
        dict(ray_dirs=f32(6, 3), A=A, trans=TRANS, ws_cl=WS_CL, packed=packed("sdf"), frame_of_ray=i32(6),
             out_sdf=f32(6, 8)), "A:0 ws_cl:0 ws_cl:1 ws_cl:2", conv="ray_dirs A trans frame_of_ray"),
    row("interp2x_boundary3d_forward", lambda o: ops.interp2x_boundary3d_forward(o["input"], 0.5),
        dict(input=f32(1, 2, 3, 4, 5)), "input:0 input:1 input:2 input:3 input:4"),
    row("interp2x_boundary3d_backward", lambda o: ops.interp2x_boundary3d_backward(o["grad_output"]),
        dict(grad_output=f32(1, 2, 5, 7, 9)), "grad_output:0 grad_output:1 grad_output:2 grad_output:3 grad_output:4"),
    row("c2f_todo_mask", lambda o: ops.c2f_todo_mask(o["is_boundary"], o["done"]),
        dict(is_boundary=bool_(3, 4, 5), done=bool_(3, 4, 5))),
    row("fragment_decode", lambda o: ops.fragment_decode(o["pix_to_face"], o["bary"], o["verts"], o["faces"], o["mask"]),
        dict(pix_to_face=i64(2, 3, 4, 2), bary=f32(2, 3, 4, 2, 3), verts=f32(5, 3), faces=i64(4, 3), mask=f32(2, 3, 4)),
        "verts:0 faces:0", conv="pix_to_face bary verts faces mask"),
    row("rasterize_meshes", lambda o: ops.rasterize_meshes(o["verts"], o["faces"], o["cameras"], 8, 8),
        dict(verts=f32(2, 5, 3), faces=i64(4, 3), cameras=f32(2, 16)), "verts:1 faces:0"),
    row("zbuf_probe",
        lambda o: ops.zbuf_probe(o["verts"], o["faces"], o["cameras"], 8, 8, o["screen_pts"], o["norm_size"], o["fill"]),
        dict(verts=f32(2, 5, 3), faces=i64(4, 3), cameras=f32(2, 16), screen_pts=f32(2, 7, 3), norm_size=f32(2, 2),
             fill=f32(2)), "verts:1 faces:0 screen_pts:1 screen_pts:2"),
    row("rasterize_points", lambda o: ops.rasterize_points(o["points"], o["features"], 8, 8, 0.1, 4),
        dict(points=f32(2, 6, 3), features=f32(2, 6))),
    row("rasterize_points_backward",
        lambda o: ops.rasterize_points_backward(o["grad_images"], o["ws"], 0, 2, 6, 8, 8, 0.1, 4),
        dict(grad_images=f32(1, 2, 8, 8), ws=torch.zeros((16,), dtype=torch.uint8)), "ws:0", conv="grad_images"),
    row("vertex_normals", lambda o: ops.vertex_normals(o["verts"], o["faces"]),
        dict(verts=f32(2, 5, 3), faces=i64(4, 3)), "verts:0 verts:1 faces:0"),
    row("surface_sample", lambda o: ops.surface_sample(o["verts"], o["faces"], 10, 0),
        dict(verts=f32(2, 5, 3), faces=i64(4, 3)), "verts:0 verts:1 faces:0"),
    row("train_rays_sample",
        lambda o: ops.train_rays_sample([o["batch[0]"]], [o["row[0]"]], [o["col[0]"]], [o["init_pts[0]"]],
                                        [o["masks[0]"]], o["camera"], 10, 0),
        {"batch[0]": i64(6), "row[0]": i64(6), "col[0]": i64(6), "init_pts[0]": f32(6, 3), "masks[0]": f32(2, 3, 4),
         "camera": f32(16)}, "masks[0]:0 masks[0]:1 masks[0]:2 camera:0"),
    row("loss_points_sample",
        lambda o: ops.loss_points_sample([o["init_pts[0]"]], [o["verts[0]"]], [o["check[0]"]], [o["batch[0]"]],
                                         [o["row[0]"]], [o["col[0]"]], [o["rays[0]"]], 16, 0),
        {"init_pts[0]": f32(6, 3), "verts[0]": f32(5, 3), "check[0]": bool_(6), "batch[0]": i64(6), "row[0]": i64(6),
         "col[0]": i64(6), "rays[0]": f32(6, 3)}, "verts[0]:0"),
    row("color_frame_mean",
        lambda o: ops.ColorFrameMeanFunction.apply(o["colors"], o["gtCs"], o["batch"], o["row"], o["col"], 2),
        dict(colors=f32(6, 3), gtCs=f32(2, 3, 4, 3), batch=i64(6), row=i64(6), col=i64(6)), "gtCs:1 gtCs:2",
        cont="colors gtCs", covers="ColorFrameMeanFunction"),
    row("normal_frame_mean",
        lambda o: ops.NormalFrameMeanFunction.apply(o["gtn"], o["J"], o["nx"], o["w"], o["batch"], 2),
        dict(gtn=f32(6, 3), J=f32(6, 3, 3), nx=f32(6, 3), w=f32(6), batch=i64(6)), cont="gtn J nx w",
        covers="NormalFrameMeanFunction"),
    row("mask_iou", lambda o: ops.mask_iou([o["masks[0]"]], [o["gt_masks[0]"]], 1),
        {"masks[0]": f32(2, 3, 4), "gt_masks[0]": f32(2, 3, 4)}),
    row("mask_iou_backward", lambda o: ops.mask_iou_backward([o["masks[0]"]], [o["mgt[0]"]], o["iu"], o["grad_loss"]),
        {"masks[0]": f32(2, 3, 4), "mgt[0]": f32(2, 3, 4), "iu": torch.zeros((1, 2, 2), dtype=torch.float64),
         "grad_loss": f32(1)}, "grad_loss:0", conv="grad_loss"),
    row("curve_fit", lambda o: ops.curve_fit(*[o[k] for k in ("center", "dirs", "init_scale", "nx", "scale", "nx_scale")]),
        dict(center=f32(3, 1, 3), dirs=f32(3, 5, 3), init_scale=f32(3, 5, 1), nx=f32(3, 1, 3), scale=f32(3, 5, 1),
             nx_scale=f32(3, 5, 1))),
    row("curve_fit_backward",
        lambda o: ops.curve_fit_backward(*[o[k] for k in ("center", "dirs", "init_scale", "nx", "scale", "nx_scale",
                                                          "dv", "dreg")]),
        dict(center=f32(3, 1, 3), dirs=f32(3, 5, 3), init_scale=f32(3, 5, 1), nx=f32(3, 1, 3), scale=f32(3, 5, 1),
             nx_scale=f32(3, 5, 1), dv=f32(3, 5, 3), dreg=f32(3, 2)), conv="dv dreg"),
    row("curve_project",
        lambda o: ops.curve_project(o["X"], o["cams"], 8, 8, [(0, 1, 0)], [0.5], 2, o["fl_masks"], o["body"]),
        dict(X=f32(6, 3), cams=f32(2, 16), fl_masks=f32(2, 4), body=f32(6)), "fl_masks:1"),
    row("curve_project_backward", lambda o: ops.curve_project_backward(o["X"], o["cams"], 1, 3, o["slot"], o["dclouds"]),
        dict(X=f32(6, 3), cams=f32(2, 16), slot=i32(6), dclouds=f32(2, 3, 2)), conv="dclouds"),
    row("shade_phong",
        lambda o: ops.shade_phong((o["pix_to_face"], None, o["bary_coords"]), o["verts"], o["normals"], o["colors"],
                                  o["faces"], o["params"]),
        dict(pix_to_face=i64(2, 3, 4, 1), bary_coords=f32(2, 3, 4, 1, 3), verts=f32(2, 5, 3), normals=f32(2, 5, 3),
             colors=f32(2, 5, 3), faces=i64(4, 3), params=f32(2, ops.SHADE_PARAMS)), "faces:0"),
    row("knn_nearest", lambda o: ops.knn_nearest(o["p1"], o["p2"], o["lengths1"], o["lengths2"]),
        dict(p1=f32(2, 5, 3), p2=f32(2, 6, 3), lengths1=i64(2), lengths2=i64(2)), "p1:1 p2:1"),
    row("knn_nearest_backward", lambda o: ops.knn_nearest_backward(o["p1"], o["p2"], o["idx"], o["grad_dists"]),
        dict(p1=f32(2, 5, 3), p2=f32(2, 6, 3), idx=i64(2, 5), grad_dists=f32(2, 5)), "p2:1", conv="grad_dists"),
    row("mesh_adjacency", lambda o: ops.mesh_adjacency(o["faces"], 5), dict(faces=i64(4, 3)), "faces:0"),
    row("nricp_warp", lambda o: ops.nricp_warp(o["X"], o["x"], o["normals"]),
        dict(X=f32(5, 3, 4), x=f32(5, 3), normals=f32(5, 3))),
    row("nricp_step",
        lambda o: ops.nricp_step(o["x"], o["normals"], o["target_v"], o["target_n"], o["corr_idx"],
                                 (o["row_ptr"], o["col"], None, o["boundary"]), o["X"],
                                 (o["exp_avg"], o["exp_avg_sq"], o["max_exp_avg_sq"]), 1, 1.0, 1.0, stats=o["stats"]),
        dict(x=f32(5, 3), normals=f32(5, 3), target_v=f32(7, 3), target_n=f32(7, 3), corr_idx=i64(5), row_ptr=i32(6),
             col=i32(24), boundary=bool_(5), X=f32(5, 3, 4), exp_avg=f32(5, 3, 4), exp_avg_sq=f32(5, 3, 4),
             max_exp_avg_sq=f32(5, 3, 4), stats=f32(ops.NRICP_STATS)), "col:0"),
    row("laplacian_edit",
        lambda o: ops.laplacian_edit(o["verts"], (o["row_ptr"], o["col"], o["deg"], None), o["cidx"], o["ctgt"],
                                     stats=o["stats"]),
        dict(verts=f32(5, 3), row_ptr=i32(6), col=i32(24), deg=i32(5), cidx=i64(3), ctgt=f32(3, 3),
             stats=f32(ops.LAP_EDIT_STATS)), "col:0"),
    row("surface_solve",
        lambda o: ops.surface_solve(torch.zeros(3), o["rays"], o["seeds"], o["batch_inds"], o["sdf_packed"], None,
                                    o["tr_packed"], None, o["conds"], (o["A"], o["trans"], o["ws_cl"], *BOX), 1e-4, 5.0,
                                    1.0, 1.0, 2),
        dict(rays=f32(6, 3), seeds=f32(6, 3), batch_inds=i64(6), sdf_packed=packed("sdf"),
             tr_packed=packed("translator"), conds=f32(2, 128), A=A, trans=TRANS, ws_cl=WS_CL),
        "ws_cl:0 ws_cl:1 ws_cl:2", conv="rays seeds batch_inds conds A trans"),
    row("surface_grad_coeffs",
        lambda o: ops.surface_grad_coeffs(o["grad_l_p"], o["grad_f_p"], o["jac"], o["rays"], o["d_minus_c"]),
        dict(grad_l_p=f32(6, 3), grad_f_p=f32(6, 3), jac=f32(6, 3, 3), rays=f32(6, 3), d_minus_c=f32(6, 3)),
        conv="grad_l_p grad_f_p jac rays d_minus_c"),
    row("implicit_surface_grad",
        lambda o: ops.implicit_surface_grad(o["grad_l_p"], o["grad_f_p"], o["jac"], o["rays"], o["d"], [0, 6],
                                            o["cam_pos"], want_ray_grad=True),
        dict(grad_l_p=f32(6, 3), grad_f_p=f32(6, 3), jac=f32(6, 3, 3), rays=f32(6, 3), d=f32(6, 3), cam_pos=f32(3))),
    row("svd3x3", lambda o: ops.Svd3x3Function.apply(o["J"]), dict(J=f32(4, 3, 3)), "J:0", covers="Svd3x3Function",
        shape_error=TypeError),
]

# operands that ops.py allocates itself, on the per-layer training path
EXEMPT = {"pe_forward", "split_planes", "weight_planes", "pe_forward_planes", "mlp_layer_planes", "mlp_wgrad_planes",
          "colsum", "softplus_tangent_planes", "add_split_planes", "pe_backward", "sdf_reverse_chain",
          "plain_reverse_chain", "C2fLevel", "read_c2f_levels"}

WRONG_DTYPE = {torch.float32: torch.float16, torch.float64: torch.float16, torch.int64: torch.int32,
               torch.int32: torch.int64, torch.bool: torch.uint8, torch.uint8: torch.bool}


def _strided(t):
    """A non-contiguous view with t's shape and dtype (one axis of extent > 1 read at stride 2)."""
    d = next(i for i, n in enumerate(t.shape) if n > 1)
    s = list(t.shape)
    s[d] *= 2
    return torch.zeros(s, dtype=t.dtype)[(slice(None),) * d + (slice(None, None, 2),)]


@pytest.fixture(autouse=True)
def no_launch(monkeypatch):
    def refuse(name, *args):
        raise AssertionError(f"{name} was launched for a refused call")
    monkeypatch.setattr(ops, "_launch", refuse)


def _refusal(r, o, cls=RuntimeError):
    with pytest.raises(cls) as e:
        r["call"](o)
    return str(e.value)


@pytest.mark.parametrize("r", ROWS, ids=lambda r: r["fn"])
def test_valid_cpu_operands_are_refused_for_not_being_on_cuda(r):
    msg = _refusal(r, dict(r["ops"]))
    assert "CUDA" in msg
    if r["ops"]:
        assert msg.startswith(f"{r['fn']}: ") and "not a CUDA tensor" in msg, msg


def _cases(r):
    for name, t in r["ops"].items():
        if name not in r["conv"]:
            yield name, "dtype", t.to(WRONG_DTYPE[t.dtype])
        for d in range(t.dim()):
            if f"{name}:{d}" not in r["free"]:
                s = list(t.shape)
                s[d] += 1
                yield name, f"extent {d}", torch.zeros(s, dtype=t.dtype)
        if name not in r["cont"]:
            yield name, "strided", _strided(t)


@pytest.mark.parametrize("r", ROWS, ids=lambda r: r["fn"])
def test_each_bad_operand_is_refused_by_name(r):
    for name, what, bad in _cases(r):
        o = dict(r["ops"], **{name: bad})
        cls = r["shape_error"] if what != "strided" else RuntimeError
        msg = _refusal(r, o, cls)
        if cls is not RuntimeError:
            continue
        assert msg.startswith(f"{r['fn']}: ") and "not a CUDA tensor" not in msg, (name, what, msg)
        assert msg.startswith(f"{r['fn']}: {name} must be") or re.search(rf"from {re.escape(name)}[,)]", msg), \
            (name, what, msg)
        if what == "strided":
            assert "contiguous" in msg, msg


def _launching_functions():
    """Top-level functions and autograd.Function forwards / classes of ops.py that call _launch themselves.  A
    Function's backward receives cotangents autograd shapes like the forward's outputs, with tensors the forward
    checked and saved."""
    tree = ast.parse(inspect.getsource(ops))

    def launches(node):
        return any(isinstance(n, ast.Call) and getattr(n.func, "id", None) == "_launch" for n in ast.walk(node))
    names = set()
    for node in tree.body:
        if isinstance(node, ast.FunctionDef) and launches(node):
            names.add(node.name)
        elif isinstance(node, ast.ClassDef):
            if any(isinstance(m, ast.FunctionDef) and m.name != "backward" and launches(m) for m in node.body):
                names.add(node.name)
    return names


def test_every_launching_wrapper_has_a_row():
    covered = set().union(*(r["covers"] for r in ROWS))
    missing = _launching_functions() - EXEMPT - covered
    assert not missing, sorted(missing)
