"""The fused tensor-core engine (`sdf_tc_kernel`, csrc/sdf_mlp_tc.cu) across multi-wave launches, ragged tails and output
bounds, for all ten instantiations <kJvp, kNet, kPasses> and the fp32 SIMT kernel on the same entries:

    SDF points          <false, 0, *>   ops.sdf_mlp_forward (with and without features), SIMT too
    SDF render          <false, 0, *>   ops.render_sdf (inverse LBS in the prologue, first hit after), SIMT too
    SDF forward mode    <true, 0, *>    ops.sdf_value_and_grad (with and without features)
    translator (+LBS)   <false, 1, *>   ops.deformer_forward
    translator Jacobian <true, 1, *>    ops.deformer_forward(want_jacobian=True), with and without LBS
    colour              <false, 2, *>   ops.rendernet_forward

The grid is min(tiles, SMs), so a CTA runs more than one tile only when the launch has more tiles than the device has SMs.
The ring slots and phases, the kBarPeReady / kBarPeFree parities, the double-buffered valid flags and the prologue
writing tile it+1's input while tile it computes all carry state from one tile to the next.  Every size here is derived
from the SM count S and the points per tile ppt (64, or 16 in forward mode): 1, ppt-1, ppt+1, S ppt (one full wave),
S ppt + 1 (CTA 0 runs a second tile of one row), 3 S ppt + r (every CTA runs at least three tiles, both barrier parities)
and, for the bit-exact checks, 10 S ppt + r.  The render path evaluates SAMPLES samples per ray, so its sizes are rounded
up to whole rays; the tile counts asserted below are those of the rounded sizes.

Three kinds of checks:
  * position invariance, bit-exact: a multi-wave launch equals launches of at most S ppt points (one tile per CTA), and a
    permuted batch gives the permuted outputs.  Every output element depends only on its own row (its own 4-row group in
    forward mode) and its MMAs run in a fixed order, so any difference means that one tile or row leaked into another.
  * accuracy against float64 (oracle/oracle_torch.py on the same effective weights) on the first, the last and the
    wave-boundary tiles plus 512 random rows; the bounds are listed at ACC_BOUND.
  * output bounds: each C entry writes into buffers with a tile of NaN-pattern guard rows before and after; the guards
    must be bit-unchanged, every row in [0, P) written, and disabling an optional output must not change the others.
Plus the device-count launch (recmv_sdf_mlp_fwd_counted) and the frame selection and clamping of DESIGN.md section 6."""
import ctypes
from ctypes import byref

import pytest
import torch

from conftest import norm_err, rel_err
from oracle import oracle_torch as ot
from recmv_b200 import _lib, ops, synth, testing
from recmv_b200 import model as M

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
SIMT, TC3, TC1 = _lib.MLP_FP32_SIMT, _lib.MLP_TC_F16X3, _lib.MLP_TC_F16X1
MODE_NAME = {SIMT: "simt", TC3: "tc3", TC1: "tc1"}
RATIO = 0.35          # annealing ratio: the third PE band is partly on, so its weights reach the tangent rows
SAMPLES = 5           # render: samples per ray (odd, so rays straddle tile boundaries)
NUM_FRAMES = 3
GUARD = 64            # guard rows before and after every output (at least one tile)
NAN_BITS = 0x7FBADBAD  # a NaN bit pattern no kernel writes

# Accuracy against float64.  sdf / feat: element-wise |a-b| / max(|b|, 1e-2) (the project's bar, F64_BOUND in
# test_gpu_sdf.py); every other output: max |a-b| / rms(truth) (norm_err), since offsets, gradients and Jacobian entries
# cross zero at no natural scale.  The render sdf is compared at the kernel's own x_c (x_c has its own row).  Measured
# on an H100 80GB HBM3 (400 W power limit), maximum over every size and variant of this file (the inputs are seeded):
#   simt  sdf 5.0e-5  feat 8.9e-5  xc 1.6e-6
#   tc3   sdf 7.5e-5  feat 8.7e-5  grad 6.7e-6  xc 1.6e-6  translated 7.1e-8  offset 5.0e-6  posed 6.1e-7  jac 4.4e-5
#         rgb 3.1e-6
#   tc1   sdf 1.8e-2  feat 2.0e-2  grad 1.0e-3  xc 1.6e-6  translated 3.2e-6  offset 1.9e-3  posed 4.2e-6  jac 1.6e-4
#         rgb 6.4e-4
# sdf / feat of simt and tc3 keep the project's 1.2e-4; every other bound is about 3x the measured maximum.  tc1
# (fp16 operands, not parity grade) has its own bounds.
ACC_BOUND = {
    "simt": {"sdf": 1.2e-4, "feat": 1.2e-4, "xc": 5e-6},
    "tc3": {"sdf": 1.2e-4, "feat": 1.2e-4, "grad": 2e-5, "xc": 5e-6, "translated": 3e-7, "offset": 1.5e-5, "posed": 2e-6,
            "jac": 1.5e-4, "rgb": 1e-5},
    "tc1": {"sdf": 5e-2, "feat": 5e-2, "grad": 3e-3, "xc": 5e-6, "translated": 1e-5, "offset": 5e-3, "posed": 1.5e-5,
            "jac": 5e-4, "rgb": 2e-3},
}
ELEMENTWISE = ("sdf", "feat")


@pytest.fixture(autouse=True)
def _no_aborted_launch():
    yield
    torch.cuda.synchronize()
    ops.check_async_errors()  # every mbarrier wait in the tensor-core kernel is bounded; none may have timed out


# ---------------------------------------------------------------------------------------------------------------------
# the variants
# ---------------------------------------------------------------------------------------------------------------------
class Variant:
    def __init__(self, name, kind, mode, feat=True, skin=False, jac=False):
        self.name, self.kind, self.mode, self.feat, self.skin, self.jac = name, kind, mode, feat, skin, jac
        self.fwd_mode = kind == "jvp" or jac
        self.ppt = 16 if self.fwd_mode else 64          # points per 64-row tile
        net = {"sdf": 0, "jvp": 0, "render": 0, "deformer": 1, "colour": 2}[kind]
        self.inst = "simt" if mode == SIMT else \
            f"<{'true' if self.fwd_mode else 'false'}, {net}, {3 if mode == TC3 else 1}>"

    def __repr__(self):
        return self.name


def _variants():
    out = []
    for m in (SIMT, TC3, TC1):
        out += [Variant(f"sdf+feat/{MODE_NAME[m]}", "sdf", m), Variant(f"sdf/{MODE_NAME[m]}", "sdf", m, feat=False),
                Variant(f"render/{MODE_NAME[m]}", "render", m)]
    for m in (TC3, TC1):
        n = MODE_NAME[m]
        out += [Variant(f"jvp+feat/{n}", "jvp", m), Variant(f"jvp/{n}", "jvp", m, feat=False),
                Variant(f"translator/{n}", "deformer", m), Variant(f"deformer/{n}", "deformer", m, skin=True),
                Variant(f"translator-jac/{n}", "deformer", m, jac=True),
                Variant(f"deformer-jac/{n}", "deformer", m, skin=True, jac=True),
                Variant(f"colour/{n}", "colour", m)]
    return out


VARIANTS = _variants()
BY_NAME = {v.name: v for v in VARIANTS}
DEFORMERS = [v.name for v in VARIANTS if v.kind == "deformer"]
RENDERS = [v.name for v in VARIANTS if v.kind == "render"]


def test_every_tensor_core_instantiation_is_covered():
    insts = {v.inst for v in VARIANTS}
    assert insts == {"simt"} | {f"<{j}, {n}, {p}>" for j, n in (("false", 0), ("true", 0), ("false", 1), ("true", 1),
                                                                  ("false", 2)) for p in (3, 1)}


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _size(tag, ppt):
    w = _sms() * ppt
    return {"1": 1, "ppt-1": ppt - 1, "ppt+1": ppt + 1, "wave": w, "wave+1": w + 1,
            "3wave+r": 3 * w + ppt // 2 + 5, "10wave+r": 10 * w + ppt - 5}[tag]


SIZES = ["1", "ppt-1", "ppt+1", "wave", "wave+1", "3wave+r"]
MULTI_WAVE = ["3wave+r", "10wave+r"]


# ---------------------------------------------------------------------------------------------------------------------
# one scene: SDF, translator and colour networks, skinning voxel, NUM_FRAMES frames of bones and conditions
# ---------------------------------------------------------------------------------------------------------------------
_SCENE = {}


def _scene():
    if _SCENE:
        return _SCENE
    sc = _SCENE
    net = testing.build_sdf(M.getTmpSdf, seed=0, perturb_seed=101).to(DEV)
    with torch.no_grad():
        Ws, bs = net.effective_weights()
        Ws, bs = [w.detach().float().contiguous() for w in Ws], [b.detach().float().contiguous() for b in bs]
    sc["sdf_packed"] = ops.sdf_pack_weights(Ws, bs)
    sc["sdf_w64"] = ([w.cpu().double() for w in Ws], [b.cpu().double() for b in bs])
    sc["sdf_pe"] = ot.annealing_weights(6, RATIO)

    torch.manual_seed(1)
    tr = testing.perturb_module(M.MLPTranslator(128, 6), 202, scale=0.5).to(DEV)
    Ws = [getattr(tr, f"lin{l}").weight.detach().float().contiguous() for l in range(5)]
    bs = [getattr(tr, f"lin{l}").bias.detach().float().contiguous() for l in range(5)]
    sc["tr_packed"] = ops.translator_pack_weights(Ws, bs)
    sc["tr_w64"] = ([w.cpu().double() for w in Ws], [b.cpu().double() for b in bs])
    sc["tr_pe"] = ot.annealing_weights(6, RATIO)

    torch.manual_seed(2)
    rn = testing.perturb_module(M.RenderingNetwork_view_norm(256, d_in=9, d_out=3, dims=[512] * 4, mode="idr",
                                                             weight_norm=True, multires_v=4, multires_n=0), 303, scale=0.1)
    with torch.no_grad():
        Ws, bs = [], []
        for l in range(5):
            lin = getattr(rn, f"lin{l}")
            Ws.append(ot.weight_norm_effective(lin.weight_g, lin.weight_v).float().contiguous().to(DEV))
            bs.append(lin.bias.detach().float().contiguous().to(DEV))
    sc["rgb_packed"] = ops.rendernet_pack_weights(Ws, bs)
    sc["rgb_w64"] = ([w.cpu().double() for w in Ws], [b.cpu().double() for b in bs])
    sc["rgb_pe"] = ot.annealing_weights(4, RATIO)

    Js, parents, init = synth.skeleton()
    ws = synth.skinning_voxel((17, 33, 21), seed=7)
    sk = M.LBSkinner(ws, [-1.1] * 3, [1.1] * 3, Js, parents, init_pose=init, bbox_extend=torch.tensor(synth.BBOX_EXTEND),
                     bbox_center=torch.tensor(synth.BBOX_CENTER)).to(DEV)
    poses, trans = synth.poses_trans(NUM_FRAMES, seed=11)
    with torch.no_grad():
        A = sk.bone_matrices(poses.to(DEV)).contiguous()
        # the last frame shrinks the upper body's bones: where their skinning weights dominate, the blended 3x3 has
        # |det| < 1e-4 and the inverse warp is singular, so a render mixes valid samples with invalid ones (~1 %), and
        # the valid flags the prologue hands to the epilogue matter
        A[NUM_FRAMES - 1, 12:, :3, :3] *= 0.02
        t = (trans.to(DEV) + sk.extra_trans).contiguous()
    center, extend = sk.bbox_host()
    sc["skin"] = (A, t, sk.ws_channels_last(), center, extend)
    sc["skin64"] = (A.cpu().double(), t.cpu().double(), sk.ws.cpu().double(),
                    torch.tensor(center, dtype=torch.float64), float(extend))
    g = torch.Generator().manual_seed(5)
    sc["conds"] = (torch.randn((NUM_FRAMES, 128), generator=g) * 0.5).to(DEV)
    return sc


def _skin_frames(sc, F):
    A, t, ws_cl, center, extend = sc["skin"]
    return (A[:F].contiguous(), t[:F].contiguous(), ws_cl, center, extend)


# ---------------------------------------------------------------------------------------------------------------------
# inputs, launches through the public entries, and row selection
# ---------------------------------------------------------------------------------------------------------------------
ROW_KEYS = {"sdf": ("x",), "jvp": ("x",), "render": ("dirs", "fr"), "deformer": ("ps", "bi"),
            "colour": ("p", "nrm", "vd", "feat")}


def _inputs(v, n, seed):
    """Inputs of n points (render: ceil(n / SAMPLES) rays)."""
    g = torch.Generator().manual_seed(seed)
    box = lambda k: torch.rand((k, 3), generator=g) * 1.6 - 0.8  # noqa: E731
    unit = lambda k: torch.nn.functional.normalize(torch.randn((k, 3), generator=g), dim=1)  # noqa: E731
    if v.kind in ("sdf", "jvp"):
        inp = {"x": box(n)}
    elif v.kind == "render":
        R = -(-n // SAMPLES)
        uv = torch.rand((R, 2), generator=g) * 0.8 - 0.4
        inp = {"dirs": torch.nn.functional.normalize(torch.cat([uv, torch.ones((R, 1))], 1), dim=1),
               "fr": torch.randint(0, NUM_FRAMES, (R,), generator=g, dtype=torch.int32)}
    elif v.kind == "deformer":
        inp = {"ps": box(n), "bi": torch.randint(0, NUM_FRAMES, (n,), generator=g)}
    else:
        inp = {"p": box(n), "nrm": unit(n), "vd": unit(n), "feat": torch.randn((n, 256), generator=g) * 0.3}
    return {k: t.to(DEV).contiguous() for k, t in inp.items()}


def _units(v, inp):
    return inp[ROW_KEYS[v.kind][0]].shape[0]


def _points(v, inp):
    """Rows the engine sees: points, or ray samples in the render path."""
    return _units(v, inp) * (SAMPLES if v.kind == "render" else 1)


def _take(v, inp, idx):
    return {k: (t[idx].contiguous() if k in ROW_KEYS[v.kind] else t) for k, t in inp.items()}


def _run(v, inp, frames=None, want_xc=True, want_hit=True, want_offset=True, want_translated=True, **kw):
    """Every output of one launch through the public entry, as {name: tensor} (rows = points, or rays)."""
    sc = _scene()
    if v.kind == "sdf":
        sdf, feat = ops.sdf_mlp_forward(inp["x"], sc["sdf_packed"], sc["sdf_pe"], v.mode, want_feat=v.feat)
        return {"sdf": sdf, "feat": feat} if v.feat else {"sdf": sdf}
    if v.kind == "jvp":
        sdf, grad, feat = ops.sdf_value_and_grad(inp["x"], sc["sdf_packed"], sc["sdf_pe"], v.mode, want_feat=v.feat)
        return dict({"sdf": sdf, "grad": grad}, **({"feat": feat} if v.feat else {}))
    if v.kind == "render":
        A, t, ws_cl, center, extend = _skin_frames(sc, frames or NUM_FRAMES)
        fr = kw.get("frame_of_ray", inp["fr"])
        sdf, xc, hit_idx, hit_t = ops.render_sdf(inp["dirs"], synth.CAM_POS, synth.T_NEAR, synth.T_FAR, SAMPLES, A, t,
                                                 ws_cl, center, extend, sc["sdf_packed"], sc["sdf_pe"], v.mode,
                                                 frame_of_ray=fr, rays_per_frame=kw.get("rays_per_frame", 0),
                                                 want_xc=want_xc, want_hit=want_hit)
        out = {"sdf": sdf, "xc": xc, "hit_idx": hit_idx, "hit_t": hit_t}
        return {k: o for k, o in out.items() if o is not None}
    if v.kind == "deformer":
        F = frames or NUM_FRAMES
        res = ops.deformer_forward(inp["ps"], sc["conds"][:F], sc["tr_packed"], sc["tr_pe"],
                                   batch_inds=kw.get("batch_inds", inp["bi"]), points_per_frame=kw.get("ppf", 0),
                                   skin=_skin_frames(sc, F) if v.skin else None, mode=v.mode, want_offset=want_offset,
                                   want_translated=want_translated, want_jacobian=v.jac)
        out = dict(zip(("translated", "offset", "posed", "jac"), res))
        return {k: o for k, o in out.items() if o is not None}
    return {"rgb": ops.rendernet_forward(inp["p"], inp["nrm"], inp["vd"], inp["feat"], sc["rgb_packed"], sc["rgb_pe"],
                                         v.mode)}


def _tiles(v, inp):
    return -(-_points(v, inp) // v.ppt)


def _check_multi_wave(v, inp, tag):
    """The size really makes every CTA run several tiles: tiles = ceil(P / ppt) against the grid min(tiles, S)."""
    S, tiles = _sms(), _tiles(v, inp)
    min_iter = tiles // S
    assert min_iter >= (3 if tag == "3wave+r" else 10) and tiles % S != 0, (tiles, S)
    return tiles


def _assert_equal_outputs(a, b, what):
    assert a.keys() == b.keys(), what
    for k in a:
        if not torch.equal(a[k], b[k]):
            diff = (a[k] != b[k]).reshape(a[k].shape[0], -1).any(1).nonzero().view(-1)
            pytest.fail(f"{what}: output {k} differs in {diff.numel()} rows, first {diff[:8].tolist()}")


# ---------------------------------------------------------------------------------------------------------------------
# 1. position invariance, bit-exact
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("tag", MULTI_WAVE)
@pytest.mark.parametrize("name", [v.name for v in VARIANTS])
def test_multi_wave_launch_equals_one_tile_per_cta_launches(name, tag):
    v = BY_NAME[name]
    inp = _inputs(v, _size(tag, v.ppt), seed=17)
    _check_multi_wave(v, inp, tag)
    full = _run(v, inp)
    # chunks of whole tiles, at most one wave: every CTA of these launches runs exactly one tile
    S = _sms()
    chunk = 64 * (S // SAMPLES) if v.kind == "render" else S * v.ppt
    assert (chunk * (SAMPLES if v.kind == "render" else 1)) % v.ppt == 0
    n = _units(v, inp)
    parts = [_run(v, _take(v, inp, torch.arange(s, min(s + chunk, n), device=DEV))) for s in range(0, n, chunk)]
    assert len(parts) > 3
    _assert_equal_outputs(full, {k: torch.cat([p[k] for p in parts]) for k in full}, f"{name} P={_points(v, inp)}")


@pytest.mark.parametrize("tag", MULTI_WAVE)
@pytest.mark.parametrize("name", [v.name for v in VARIANTS])
def test_permuted_batch_gives_permuted_outputs(name, tag):
    """A permutation moves every point to another tile row, tile and CTA (in forward mode, its 4-row group to another
    group).  The bits must follow the point."""
    v = BY_NAME[name]
    inp = _inputs(v, _size(tag, v.ppt), seed=23)
    _check_multi_wave(v, inp, tag)
    perm = torch.randperm(_units(v, inp), generator=torch.Generator().manual_seed(29)).to(DEV)
    full = _run(v, inp)
    permuted = _run(v, _take(v, inp, perm))
    _assert_equal_outputs({k: t[perm] for k, t in full.items()}, permuted, f"{name} P={_points(v, inp)}")


# ---------------------------------------------------------------------------------------------------------------------
# 2. accuracy against float64
# ---------------------------------------------------------------------------------------------------------------------
def _sample_rows(v, inp, seed, n_random=512):
    """Units (points, or rays) of the first tile, the last tile, the tiles at the wave boundaries S-1, S, 2S, 3S, and
    n_random random ones."""
    P, ppt, S = _points(v, inp), v.ppt, _sms()
    per = SAMPLES if v.kind == "render" else 1
    tiles = -(-P // ppt)
    pts = set()
    for t in {0, tiles - 1, S - 1, S, 2 * S, 3 * S}:
        if 0 <= t < tiles:
            pts |= set(range(t * ppt, min((t + 1) * ppt, P)))
    units = {p // per for p in pts}
    n = _units(v, inp)
    k = n_random // per
    if n <= len(units) + k:
        return torch.arange(n)
    units |= set(torch.randint(0, n, (k,), generator=torch.Generator().manual_seed(seed)).tolist())
    return torch.tensor(sorted(units))


def _truth(v, inp, out, rows):
    """float64 values of the outputs on `rows` (CPU), from the oracle on the same effective weights."""
    sc = _scene()
    cpu = {k: t[rows.to(t.device)].cpu() for k, t in inp.items() if k in ROW_KEYS[v.kind]}
    if v.kind in ("sdf", "jvp"):
        x = cpu["x"].double().requires_grad_(v.kind == "jvp")
        with torch.enable_grad():
            sdf, feat = ot.sdf_mlp(x, *sc["sdf_w64"], sc["sdf_pe"])
            res = {"sdf": sdf.detach(), "feat": feat.detach()}
            if v.kind == "jvp":
                res["grad"] = torch.autograd.grad(sdf.sum(), x)[0]
        return res
    if v.kind == "render":
        A, t, ws, center, extend = sc["skin64"]
        R = rows.numel()
        dt = (synth.T_FAR - synth.T_NEAR) / SAMPLES
        tk = synth.T_NEAR + (torch.arange(SAMPLES, dtype=torch.float64) + 0.5) * dt
        xo = (torch.tensor(synth.CAM_POS, dtype=torch.float64)[None, None]
              + tk[None, :, None] * cpu["dirs"].double()[:, None, :]).reshape(-1, 3)
        bi = cpu["fr"].long().clamp(0, NUM_FRAMES - 1).repeat_interleave(SAMPLES)
        xc, ok = ot.lbs_inverse(xo, A, t, ws, center, extend, bi)
        w = ot.skin_weights(ws, xo, center, extend)
        det = torch.linalg.det((w[:, :, None] * A[bi].reshape(-1, 24, 16)).sum(1).view(-1, 4, 4)[:, :3, :3])
        # the sdf at the kernel's own x_c: the MLP against float64, x_c on its own
        xc_ours = out["xc"][rows.to(DEV)].cpu().double().reshape(-1, 3)
        sdf = ot.sdf_mlp(xc_ours, *sc["sdf_w64"], sc["sdf_pe"])[0].view(R, SAMPLES)
        return {"sdf": sdf, "xc": xc.view(R, SAMPLES, 3), "ok": ok.view(R, SAMPLES), "det": det.view(R, SAMPLES)}
    if v.kind == "deformer":
        p = cpu["ps"].double().requires_grad_(v.jac)
        bi = cpu["bi"].clamp(0, NUM_FRAMES - 1)
        with torch.enable_grad():
            tr, off = ot.translator_mlp(p, sc["conds"].cpu().double()[bi], *sc["tr_w64"], sc["tr_pe"])
            res = {"translated": tr, "offset": off}
            if v.skin:
                A, t, ws, center, extend = sc["skin64"]
                res["posed"] = ot.lbs_forward(tr, A, t, ws, center, extend, bi)
            if v.jac:
                last = res["posed"] if v.skin else tr
                res["jac"] = torch.stack([torch.autograd.grad(last[:, i].sum(), p, retain_graph=True)[0]
                                          for i in range(3)], 1)      # [n, i, j] = d out_i / d p_j
        return {k: t.detach() for k, t in res.items()}
    return {"rgb": ot.render_mlp(cpu["p"].double(), cpu["nrm"].double(), cpu["vd"].double(), cpu["feat"].double(),
                                 *sc["rgb_w64"], sc["rgb_pe"])}


def _first_hit(sdf):
    """(hit_idx, hit_t) by the stated rule from the kernel's own sdf rows [R, SAMPLES] (float64 depth)."""
    s = sdf.double()
    neg = s <= 0
    first = torch.where(neg.any(1), neg.long().argmax(1), torch.full((s.shape[0],), -1))
    first = torch.where(first > 0, first, torch.full_like(first, -1))
    k = first.clamp_min(1)
    s0, s1 = s.gather(1, (k - 1)[:, None])[:, 0], s.gather(1, k[:, None])[:, 0]
    dt = (synth.T_FAR - synth.T_NEAR) / SAMPLES
    t = synth.T_NEAR + ((k - 1).double() + 0.5) * dt + dt * s0 / (s0 - s1)
    return first, torch.where(first > 0, t, torch.zeros_like(t))


@pytest.mark.parametrize("tag", SIZES)
@pytest.mark.parametrize("name", [v.name for v in VARIANTS])
def test_accuracy_against_float64(name, tag):
    v = BY_NAME[name]
    inp = _inputs(v, _size(tag, v.ppt), seed=31)
    out = _run(v, inp)
    rows = _sample_rows(v, inp, seed=37)
    truth = _truth(v, inp, out, rows)
    ours = {k: o[rows.to(o.device)].cpu() for k, o in out.items()}
    mode = MODE_NAME[v.mode]
    errs = {}
    if v.kind == "render":
        ok, det = truth.pop("ok"), truth.pop("det")
        valid = ours["sdf"] != 1e10                      # kInvalidSdf: singular inverse warp
        assert torch.equal(valid, ok), f"{name}: validity flags differ from the float64 inverse warp"
        assert valid.float().mean() > 0.9
        assert _points(v, inp) < 8000 or bool((out["sdf"] == 1e10).any()), f"{name}: no invalid sample in the launch"
        # x_c where the blended 3x3 is well conditioned: just above the singular threshold (|det| 1e-4) the inverse
        # amplifies fp32 rounding by ~1 / |det| (measured 5.8e-6 there)
        good = ok & (det.abs() > 1e-2)
        errs["xc"] = norm_err(ours["xc"][good], truth["xc"][good])
        errs["sdf"] = rel_err(ours["sdf"][ok], truth["sdf"][ok], 1e-2)
        # first hit: index exact and depth by the stated formula, on every ray of the launch
        hi, ht = _first_hit(out["sdf"].cpu())
        assert torch.equal(out["hit_idx"].cpu().long(), hi), name
        assert (out["hit_t"].cpu().double() - ht).abs().max() < 1e-5, name
    else:
        for k, t in truth.items():
            if k == "feat" and k not in ours:
                continue
            o = ours[k].reshape(t.shape) if k != "sdf" else ours[k].reshape(-1)
            t = t.reshape(-1) if k == "sdf" else t
            errs[k] = rel_err(o, t, 1e-2) if k in ELEMENTWISE else norm_err(o, t)
    assert errs.keys() <= ACC_BOUND[mode].keys()
    P = _points(v, inp)
    table = "\n".join(f"{name:20s} {v.inst:15s} {tag:8s} P={P:6d} rows={rows.numel():4d} {k:10s} |ours-f64| {e:.2e}"
                      f"  (bound {ACC_BOUND[mode][k]:.1e})" for k, e in errs.items())
    print("\n" + table)
    for k, e in errs.items():
        assert e < ACC_BOUND[mode][k], table


# ---------------------------------------------------------------------------------------------------------------------
# 3. output bounds: the C entries write rows [0, P) of every output and nothing else
# ---------------------------------------------------------------------------------------------------------------------
class _Guarded:
    """Outputs inside larger buffers with GUARD rows of the NaN pattern before and after."""

    def __init__(self):
        self.bufs = {}

    def __call__(self, name, shape, dtype=torch.float32):
        full = torch.empty((GUARD + shape[0] + GUARD,) + tuple(shape[1:]), dtype=dtype, device=DEV)
        full.view(torch.int32).fill_(NAN_BITS)
        self.bufs[name] = full
        return full[GUARD:GUARD + shape[0]]

    def check(self, what):
        for name, full in self.bufs.items():
            bits = full.view(torch.int32).reshape(full.shape[0], -1)
            n = full.shape[0] - 2 * GUARD
            assert bool((bits[:GUARD] == NAN_BITS).all()), f"{what}: {name} written before row 0"
            assert bool((bits[GUARD + n:] == NAN_BITS).all()), f"{what}: {name} written at or after row P={n}"
            assert not bool((bits[GUARD:GUARD + n] == NAN_BITS).any(1).any()), f"{what}: {name} has rows not written"


def _run_raw(v, inp, alloc):
    """The same launch as _run through the C entry, with the argument marshalling of ops.py and caller-owned outputs."""
    sc = _scene()
    lib, P, p_ = _lib.load(), _units(v, inp), ops._ptr
    st = ops._stream(next(iter(inp.values())))
    out = {}
    with torch.cuda.device(DEV):
        if v.kind in ("sdf", "jvp"):
            out["sdf"] = alloc("sdf", (P, 1))
            feat = out["feat"] = alloc("feat", (P, 256)) if v.feat else None
            if v.kind == "sdf":
                s = lib.recmv_sdf_mlp_fwd(p_(inp["x"]), p_(sc["sdf_packed"]), ops._pe_array(sc["sdf_pe"]),
                                          p_(out["sdf"]), p_(feat), P, v.mode, st)
            else:
                out["grad"] = alloc("grad", (P, 3))
                s = lib.recmv_sdf_mlp_fwd_grad(p_(inp["x"]), p_(sc["sdf_packed"]), ops._pe_array(sc["sdf_pe"]),
                                               p_(out["sdf"]), p_(feat), p_(out["grad"]), P, v.mode, st)
        elif v.kind == "render":
            A, t, ws_cl, center, extend = sc["skin"]
            out.update(sdf=alloc("sdf", (P, SAMPLES)), xc=alloc("xc", (P, SAMPLES, 3)),
                       hit_idx=alloc("hit_idx", (P,), torch.int32), hit_t=alloc("hit_t", (P,)))
            rm, vox = ops.make_raymarch(synth.CAM_POS, synth.T_NEAR, synth.T_FAR, SAMPLES), ops.make_voxel(ws_cl, center,
                                                                                                          extend)
            s = lib.recmv_render_sdf(p_(inp["dirs"]), byref(rm), p_(A), p_(t), p_(inp["fr"]), 0, NUM_FRAMES, byref(vox),
                                     p_(sc["sdf_packed"]), ops._pe_array(sc["sdf_pe"]), p_(out["sdf"]), p_(out["xc"]),
                                     p_(out["hit_idx"]), p_(out["hit_t"]), P, v.mode, st)
        elif v.kind == "deformer":
            A, t, ws_cl, center, extend = sc["skin"]
            out.update(translated=alloc("translated", (P, 3)), offset=alloc("offset", (P, 3)))
            if v.skin:
                out["posed"] = alloc("posed", (P, 3))
            vox = byref(ops.make_voxel(ws_cl, center, extend)) if v.skin else None
            args = [p_(inp["ps"]), p_(sc["conds"]), p_(inp["bi"]), 0, NUM_FRAMES, p_(sc["tr_packed"]),
                    ops._pe_array(sc["tr_pe"]), p_(A) if v.skin else None, p_(t) if v.skin else None, vox,
                    p_(out["translated"]), p_(out["offset"]), p_(out.get("posed"))]
            if v.jac:
                out["jac"] = alloc("jac", (P, 3, 3))
                s = lib.recmv_deformer_fwd_jac(*args, p_(out["jac"]), P, v.mode, st)
            else:
                s = lib.recmv_deformer_fwd(*args, P, v.mode, st)
        else:
            out["rgb"] = alloc("rgb", (P, 3))
            s = lib.recmv_rendernet_fwd(p_(inp["p"]), p_(inp["nrm"]), p_(inp["vd"]), p_(inp["feat"]), p_(sc["rgb_packed"]),
                                        (ctypes.c_float * 8)(*sc["rgb_pe"]), p_(out["rgb"]), P, v.mode, st)
    _lib.check(s, f"{v.name} C entry")
    return {k: o for k, o in out.items() if o is not None}


@pytest.mark.parametrize("tag", ["ppt-1", "ppt+1", "3wave+r"])
@pytest.mark.parametrize("name", [v.name for v in VARIANTS])
def test_outputs_are_written_in_rows_0_to_P_only(name, tag):
    v = BY_NAME[name]
    inp = _inputs(v, _size(tag, v.ppt), seed=41)
    g = _Guarded()
    raw = _run_raw(v, inp, g)
    torch.cuda.synchronize()
    g.check(f"{name} P={_points(v, inp)}")
    _assert_equal_outputs(_run(v, inp), raw, f"{name}: C entry vs public entry")


@pytest.mark.parametrize("name", [v.name for v in VARIANTS if v.feat and v.kind != "colour"])
def test_disabling_an_optional_output_leaves_the_others_bit_identical(name):
    """want_feat (SDF, forward mode), want_xc / want_hit (render), want_offset / want_translated (deformer)."""
    v = BY_NAME[name]
    inp = _inputs(v, _size("3wave+r", v.ppt), seed=43)
    full = _run(v, inp)
    if v.kind in ("sdf", "jvp"):
        lean = _run(BY_NAME[name.replace("+feat", "")], inp)
        _assert_equal_outputs({k: t for k, t in full.items() if k != "feat"}, lean, f"{name} without features")
    elif v.kind == "render":
        for kw in ({"want_xc": False}, {"want_hit": False}, {"want_xc": False, "want_hit": False}):
            part = _run(v, inp, **kw)
            _assert_equal_outputs({k: full[k] for k in part}, part, f"{name} {kw}")
            assert ("xc" in part) == kw.get("want_xc", True) and ("hit_idx" in part) == kw.get("want_hit", True)
    else:
        for kw in ({"want_offset": False}, {"want_translated": False}, {"want_offset": False, "want_translated": False}):
            part = _run(v, inp, **kw)
            _assert_equal_outputs({k: full[k] for k in part}, part, f"{name} {kw}")
            assert ("offset" in part) == kw.get("want_offset", True)
            assert ("translated" in part) == kw.get("want_translated", True)


# ---------------------------------------------------------------------------------------------------------------------
# 4. the device-count launch
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("p_dev", ["0", "-5", "1", "64", "P-1", "P", "P+100"])
@pytest.mark.parametrize("mode", [TC3, TC1], ids=["tc3", "tc1"])
def test_counted_launch_evaluates_exactly_the_device_count(mode, p_dev):
    """recmv_sdf_mlp_fwd_counted sizes its grid for the capacity P and reads the point count from device memory, clamped
    to [0, P]: rows below the count equal sdf_mlp_forward on those points, the rest keep what was there."""
    sc = _scene()
    v = BY_NAME[f"sdf+feat/{MODE_NAME[mode]}"]
    P = _size("3wave+r", 64)
    inp = _inputs(v, P, seed=47)
    n_dev = {"0": 0, "-5": -5, "1": 1, "64": 64, "P-1": P - 1, "P": P, "P+100": P + 100}[p_dev]
    n = min(max(n_dev, 0), P)
    count = torch.tensor([n_dev], dtype=torch.int32, device=DEV)
    g = _Guarded()
    sdf, feat = g("sdf", (P, 1)), g("feat", (P, 256))
    with torch.cuda.device(DEV):
        _lib.check(_lib.load().recmv_sdf_mlp_fwd_counted(ops._ptr(inp["x"]), ops._ptr(sc["sdf_packed"]),
                                                         ops._pe_array(sc["sdf_pe"]), ops._ptr(sdf), ops._ptr(feat), P,
                                                         ops._ptr(count), mode, ops._stream(inp["x"])),
                   "recmv_sdf_mlp_fwd_counted")
    ref = _run(v, _take(v, inp, torch.arange(n, device=DEV)))
    torch.cuda.synchronize()
    for name, full in g.bufs.items():
        bits = full.view(torch.int32).reshape(full.shape[0], -1)
        assert bool((bits[:GUARD] == NAN_BITS).all()) and bool((bits[GUARD + n:] == NAN_BITS).all()), (name, n_dev)
        assert not bool((bits[GUARD:GUARD + n] == NAN_BITS).any()), (name, n_dev)
    assert torch.equal(sdf[:n], ref["sdf"]) and torch.equal(feat[:n], ref["feat"]), n_dev


# ---------------------------------------------------------------------------------------------------------------------
# 5. frame selection and clamping
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", DEFORMERS)
def test_deformer_frame_selection(name):
    """batch_inds = p // ppf is the same launch as points_per_frame = ppf; with one frame, batch_inds = None and
    points_per_frame = 0 select it for every point."""
    v = BY_NAME[name]
    inp = _inputs(v, _size("3wave+r", v.ppt), seed=53)
    P = _units(v, inp)
    ppf = -(-P // NUM_FRAMES)
    by_index = _run(v, inp, batch_inds=torch.arange(P, device=DEV) // ppf)
    by_count = _run(v, inp, batch_inds=None, ppf=ppf)
    _assert_equal_outputs(by_index, by_count, f"{name}: batch_inds vs points_per_frame")
    one_none = _run(v, inp, frames=1, batch_inds=None, ppf=0)
    one_zero = _run(v, inp, frames=1, batch_inds=torch.zeros(P, dtype=torch.long, device=DEV))
    _assert_equal_outputs(one_none, one_zero, f"{name}: one frame, no indices")


@pytest.mark.parametrize("name", RENDERS)
def test_render_frame_selection(name):
    v = BY_NAME[name]
    inp = _inputs(v, _size("3wave+r", v.ppt), seed=59)
    R = _units(v, inp)
    rpf = -(-R // NUM_FRAMES)
    by_index = _run(v, inp, frame_of_ray=(torch.arange(R, device=DEV) // rpf).int())
    by_count = _run(v, inp, frame_of_ray=None, rays_per_frame=rpf)
    _assert_equal_outputs(by_index, by_count, f"{name}: frame_of_ray vs rays_per_frame")


@pytest.mark.parametrize("name", DEFORMERS + RENDERS)
def test_out_of_range_frame_indices_are_clamped(name):
    """DESIGN.md section 6: indices below 0 select frame 0, indices >= F the last frame."""
    v = BY_NAME[name]
    inp = _inputs(v, _size("3wave+r", v.ppt), seed=61)
    n = _units(v, inp)
    g = torch.Generator().manual_seed(67)
    wild = torch.tensor([-1, NUM_FRAMES, NUM_FRAMES + 5, 0, NUM_FRAMES - 1])[torch.randint(0, 5, (n,), generator=g)]
    wild = wild.to(DEV)
    clamped = wild.clamp(0, NUM_FRAMES - 1)
    if v.kind == "render":
        a, b = _run(v, inp, frame_of_ray=wild.int()), _run(v, inp, frame_of_ray=clamped.int())
    else:
        a, b = _run(v, inp, batch_inds=wild), _run(v, inp, batch_inds=clamped)
    _assert_equal_outputs(a, b, f"{name}: out-of-range frame indices")
