#!/usr/bin/env python
"""K6 attribution: where a block's cycles go in intra_block, on the bench's I picture (intra_ctu_kernel) and one B picture (intra_kernel).

For every library given it runs both pictures (flattened by DecLibReconB200's host stages through helpers.SeamCase, as bench.py builds them) and prints
  * K6 device time per picture (CUDA events around the K6 launches), the depth of the picture's intra list (tools/intra_depth.py) and us per level;
  * for a library built with -DB200_K6_PHASES: the cycles per block of each phase of intra_block (wait, reference fill, reference filter, prediction and
    store, publish), luma and chroma, for the kernel that ran.
The counters' atomics add a little to each block: compare phase tables of attribution builds, and times of default builds.

usage (GPU): python tools/k6_phases.py [--lib PATH ...] [--runs N] [bench workload options]
Without --lib the tool builds the attribution library from the tree into a temporary directory and measures that."""
import os, sys, json, argparse, subprocess, tempfile, ctypes as C
import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tools"))
from vvdec_b200 import abi, bindings
import intra_depth

PHASES = ["wait", "fill", "filter", "predict+store", "publish"]
KERNELS = ["intra_kernel", "intra_ctu_kernel"]


def build_attribution(out_dir):
    subprocess.check_call(["make", "-C", os.path.join(ROOT, "vvdec_b200", "csrc"), "-j8", "-s", f"OUT={out_dir}/", "DEFS=-DB200_K6_PHASES"])
    return os.path.join(out_dir, "libvvdec_b200.so")


def gpu_identity():
    try:
        return subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=10).stdout.strip()
    except Exception:
        return "unknown"


def measure(path, wl, pics, depths, runs):
    lib = C.CDLL(path); bindings.declare(lib)
    def check(rc):
        if rc != 0: raise RuntimeError(f"{path}: error {rc}: {lib.b200_last_error().decode()}")
    phases = getattr(lib, "b200_k6_phases", None)
    if phases: phases.argtypes = [C.POINTER(C.c_ulonglong), C.c_int]
    g = abi.make_geom(wl.args.width, wl.args.height, 10)
    ctx = C.c_void_p(); check(lib.b200_ctx_create(C.byref(ctx), C.byref(g), 6, 2, 0))
    res = {"lib": path, "pictures": {}}
    try:
        for s in range(6): check(lib.b200_ctx_load_slot(ctx, s, abi.plane_ptrs(wl.base.refs[s % 4])))
        cnt = (C.c_ulonglong * 24)()
        for name, pic in pics:
            h = lib.b200_pic_upload(ctx, C.byref(pic["struct"])); assert h >= 0, lib.b200_last_error()
            for _ in range(3): check(lib.b200_pic_run(ctx, h))
            if phases: check(phases(cnt, 1))
            check(lib.b200_ctx_set_profiling(ctx, 1))
            for _ in range(runs): check(lib.b200_pic_run(ctx, h))
            kms = (C.c_float * 10)(); kn = (C.c_int * 10)()
            check(lib.b200_ctx_get_kernel_ms_n(ctx, kms, kn, 10)); check(lib.b200_ctx_set_profiling(ctx, 0))
            k6 = kms[8] / runs
            r = {"k6_ms": round(k6, 4), "depth": depths[name]["depth"], "us_per_level": round(1e3 * k6 / max(1, depths[name]["depth"]), 3)}
            if phases:
                check(phases(cnt, 1))
                a = np.array(cnt[:], np.float64).reshape(2, 2, 6)
                for kern in range(2):
                    for ch, chn in enumerate(("luma", "chroma")):
                        if a[kern, ch, 5] > 0:
                            r[f"{KERNELS[kern]}.{chn}"] = {"blocks": int(a[kern, ch, 5] / runs), **{p: round(a[kern, ch, i] / a[kern, ch, 5]) for i, p in enumerate(PHASES)}}
            res["pictures"][name] = r
    finally:
        lib.b200_ctx_destroy(ctx)
    return res


def main():
    ap = argparse.ArgumentParser()
    intra_depth.add_args(ap)
    ap.add_argument("--lib", action="append", help="library to measure (repeatable); default: an attribution build of the tree")
    ap.add_argument("--runs", type=int, default=10, help="timed runs of each picture")
    args = ap.parse_args()
    args.b_pictures = 1
    tmp = None
    libs = args.lib
    if not libs:
        tmp = tempfile.TemporaryDirectory(prefix="k6_phases_")
        libs = [build_attribution(tmp.name)]
    wl, pics = intra_depth.bench_pictures(args)
    depths = {name: intra_depth.depth(pic["intraTus"], args.width, args.height) for name, pic in pics}
    print("gpu:", gpu_identity())
    print("depth:", json.dumps(depths))
    for path in libs:
        r = measure(path, wl, pics, depths, args.runs)
        print(f"\n{path}")
        for name, p in r["pictures"].items():
            print(f"  {name} picture: K6 {p['k6_ms']:.4f} ms, depth {p['depth']}, {p['us_per_level']:.3f} us per level")
            rows = [(k, v) for k, v in p.items() if isinstance(v, dict)]
            if rows:
                print(f"    {'kernel.channel':24} {'blocks':>7} " + " ".join(f"{ph:>13}" for ph in PHASES) + f" {'total':>7}")
                for k, v in rows:
                    print(f"    {k:24} {v['blocks']:7d} " + " ".join(f"{v[ph]:13d}" for ph in PHASES) + f" {sum(v[ph] for ph in PHASES):7d}")
        print("json:", json.dumps(r), flush=True)
    if tmp: tmp.cleanup()


if __name__ == "__main__":
    main()
