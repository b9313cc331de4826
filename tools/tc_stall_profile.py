"""Where the cycles of the fused render kernel go.

Builds the library with RECMV_TC_STALL_PROF=1 from a copy of recmv_b200/csrc in a temporary directory (the product
library and its build directory are not touched), renders one 512x512-ray x 64-sample frame of bench.py's scene per
mode and prints each stall counter of sdf_tc_kernel as a share of the cycles of its role:

  consumers (thread 0 of each MMA warpgroup): waits on FULL (weights not arrived), wgmma.wait_group (tensor pipe busy),
  epilogue, the two named barriers per layer, the wait for the tile input; what is left is issuing MMAs;
  producers (the TMA lane of each ring): waits on EMPTY (ring full).

  python tools/tc_stall_profile.py [--modes tc3,tc1] [--src CSRC_DIR] [--json OUT]

--src profiles another csrc tree (e.g. an earlier revision's, to compare); its include/ must sit at ../../include.
The counters are clock64() reads around each wait: the profiling build runs a little slower than the product.
"""
import argparse
import ctypes
import json
import os
import shutil
import subprocess
import sys
import tempfile

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

COUNTERS = ("full_wait", "wg_wait", "epilogue", "named_barriers", "pe_ready_wait", "consumer_total",
            "empty_wait", "producer_total")
CONSUMER_STALLS = ("full_wait", "wg_wait", "epilogue", "named_barriers", "pe_ready_wait")
MODES = {"tc3": 1, "tc1": 2}


def build_profiling_lib(src, tmp):
    """Copy src (a csrc directory) and its ../../include into tmp and build the profiling library there."""
    csrc = os.path.join(tmp, "recmv_b200", "csrc")
    shutil.copytree(src, csrc, ignore=shutil.ignore_patterns("build", "*.so", "*.o"))
    shutil.copytree(os.path.join(src, "..", "..", "include"), os.path.join(tmp, "include"))
    subprocess.check_call(["make", "-s", f"-j{os.cpu_count() or 8}", "-C", csrc, "EXTRA=-DRECMV_TC_STALL_PROF=1"],
                          stdout=subprocess.DEVNULL)
    return os.path.join(tmp, "recmv_b200", "librecmv_b200.so")


def card():
    q = "name,power.limit,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError) as e:
        out = f"unavailable ({e})"
    return {"torch_name": torch.cuda.get_device_name(0), "nvidia_smi": f"{q}: {out}"}


def profile_frame(lib, mode):
    from recmv_b200 import ops, synth
    from recmv_b200.render import SdfRenderer
    dev = torch.device("cuda", 0)
    ren = SdfRenderer(dev, mode=MODES[mode], samples=64)
    poses, trans = synth.poses_trans(1, seed=11, device="cpu")
    A, t = ren.bone_matrices(poses.to(dev), trans.to(dev))
    dirs = synth.pinhole_rays(512, 512, device=dev)
    counters = (ctypes.c_ulonglong * len(COUNTERS))()
    ren.render(dirs, A, t, rays_per_frame=dirs.shape[0])   # warm-up
    assert lib.recmv_tc_stall_profile(counters, len(COUNTERS), 1) == 0
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    ren.render(dirs, A, t, rays_per_frame=dirs.shape[0])
    e1.record()
    assert lib.recmv_tc_stall_profile(counters, len(COUNTERS), 1) == 0
    ops.check_async_errors()
    c = dict(zip(COUNTERS, (int(v) for v in counters)))
    ct, pt = max(c["consumer_total"], 1), max(c["producer_total"], 1)
    shares = {k: c[k] / ct for k in CONSUMER_STALLS}
    shares["issue_and_rest"] = 1.0 - sum(shares.values())
    shares["producer_empty_wait"] = c["empty_wait"] / pt
    return {"mode": mode, "frame_ms_profiling_build": e0.elapsed_time(e1), "cycles": c, "shares": shares}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--modes", default="tc3,tc1")
    ap.add_argument("--src", default=os.path.join(ROOT, "recmv_b200", "csrc"))
    ap.add_argument("--json", default=None, help="also write the results to this file")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("tc_stall_profile.py needs a CUDA device")
    with tempfile.TemporaryDirectory(prefix="recmv_stall_") as tmp:
        so = build_profiling_lib(os.path.abspath(args.src), tmp)
        from recmv_b200 import _lib
        _lib.LIB_PATH = so                       # every recmv_b200 call of this process goes to the profiling build
        lib = _lib.load()
        lib.recmv_tc_stall_profile.restype = ctypes.c_int
        lib.recmv_tc_stall_profile.argtypes = [ctypes.POINTER(ctypes.c_ulonglong), ctypes.c_int, ctypes.c_int]
        res = {"src": os.path.abspath(args.src), "card": card(), "runs": []}
        for mode in args.modes.split(","):
            r = profile_frame(lib, mode)
            res["runs"].append(r)
            s = r["shares"]
            print(f"{mode}: frame {r['frame_ms_profiling_build']:.1f} ms (profiling build); consumer cycles: "
                  + ", ".join(f"{k} {100 * s[k]:.1f}%" for k in CONSUMER_STALLS + ("issue_and_rest",))
                  + f"; producer cycles: empty_wait {100 * s['producer_empty_wait']:.1f}%")
        print("card:", res["card"])
    if args.json:
        with open(args.json, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
