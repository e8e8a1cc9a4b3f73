#!/usr/bin/env python
"""Longest dependency chain of an intra list (b200_intra_tu records in decoding order), as the K6 kernels wait on it.

A block depends on the blocks whose done word intra_block waits for: the region before it (ISP regions after the first), the owners of the units of its
corner, above and left reference samples, and for CCLM the owners of the luma units its templates and co-located block read.  The owner of a unit is the
last record of the list that writes it (intra_owner_kernel); only owners earlier in the list count.  The depth of a list is the number of blocks on its
longest chain: the K6 time of a list over its depth is the time per level (us per level), the latency of one block-to-block hop.

usage: python tools/intra_depth.py [--width W --height H --seed S --intra-pct P --isp-pct Q]   (the bench's I picture and B pictures; needs the
       compiled reference, no GPU)"""
import os, sys, argparse
import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from vvdec_b200 import abi


def depth(tus, W, H):
    """{blocks, roots (blocks that wait for none), depth (longest chain, in blocks), median_samples} of the intra list `tus` (INTRA_TU_DTYPE) of a
    W x H 4:2:0 picture."""
    n = len(tus)
    if n == 0: return {"blocks": 0, "roots": 0, "depth": 0, "median_samples": 0}
    own = [np.full((H // 4 + 1, W // 4 + 1), -1, np.int64), np.full((H // 4 + 1, W // 4 + 1), -1, np.int64), np.full((H // 4 + 1, W // 4 + 1), -1, np.int64)]
    x, y, l2w, l2h, comp = (tus[f].astype(np.int64) for f in ("x", "y", "log2w", "log2h", "comp"))
    for i in range(n):                                           # the last writer of a unit owns it (atomicMax over the list)
        c = comp[i]; ush = 1 if c else 2
        own[c][y[i] >> ush:(y[i] >> ush) + max(1, (1 << l2h[i]) >> ush), x[i] >> ush:(x[i] >> ush) + max(1, (1 << l2w[i]) >> ush)] = i
    level = np.zeros(n, np.int64)
    for i in range(n):
        t = tus[i]; c = int(comp[i]); w, h = 1 << int(l2w[i]), 1 << int(l2h[i]); ush = 1 if c else 2
        bx, by, k = int(x[i]), int(y[i]), 0
        if t["flags"] & abi.INTRA_ISP:                           # IspGeom: the CU's neighbourhood, the region before this one
            split, k = int(t["mip"]) & 3, (int(t["mip"]) >> 2) & 3
            if split == 1: by -= k * h
            else: bx -= k * w
        deps = [own[c][(by - 1) >> ush, (bx - 1) >> ush:((bx - 1) >> ush) + 1]] if (t["flags"] & abi.INTRA_AVAIL_TL) and bx > 0 and by > 0 else []
        if by > 0: deps.append(own[c][(by - 1) >> ush, bx >> ush:(bx >> ush) + int(t["numAbove"])])
        if bx > 0: deps.append(own[c][by >> ush:(by >> ush) + int(t["numLeft"]), (bx - 1) >> ush])
        if t["mode"] >= abi.INTRA_LM:
            aCu, lCu = bool(t["flags"] & abi.INTRA_LM_ABOVE), bool(t["flags"] & abi.INTRA_LM_LEFT)
            nA = max(w, (2 * int(t["lmAbove"]) if t["mode"] == abi.INTRA_MDLM_T else w) if aCu else 0)
            nL = max(h, (2 * int(t["lmLeft"]) if t["mode"] == abi.INTRA_MDLM_L else h) if lCu else 0)
            ux0, ux1 = max(0, (2 * int(x[i]) - (4 if lCu else 0)) >> 2), min(W - 1, 2 * int(x[i]) + 2 * nA - 1) >> 2
            uy0, uy1 = max(0, (2 * int(y[i]) - (4 if aCu else 0)) >> 2), min(H - 1, 2 * int(y[i]) + 2 * nL - 1) >> 2
            deps.append(own[0][uy0:uy1 + 1, ux0:ux1 + 1].ravel())
        o = np.concatenate(deps) if deps else np.zeros(0, np.int64)
        o = o[(o >= 0) & (o < i)]
        if k: o = np.append(o, i - 1)
        level[i] = 1 + (level[o].max() if len(o) else 0)
    roots = int((level == 1).sum())
    return {"blocks": n, "roots": roots, "depth": int(level.max()), "median_samples": int(np.median((1 << l2w) * (1 << l2h)))}


def bench_pictures(args):
    """The bench's I picture and B pictures, flattened by DecLibReconB200's host stages as bench.py builds them: [(name, picture dict)]."""
    import bench
    ns = argparse.Namespace(seed=args.seed, width=args.width, height=args.height, intra_pct=args.intra_pct, isp_pct=args.isp_pct, distinct=args.distinct, gop=32)
    wl = bench.Workload(ns, 0)
    out = []
    for name, case in [("I", wl.I)] + [(f"B{j}", b) for j, b in enumerate(wl.B[:args.b_pictures])]:
        pic, _ = case.flatten(threads=os.cpu_count())
        pic["struct"].dstSlot = 4
        out.append((name, pic))
    return wl, out


def add_args(ap):
    ap.add_argument("--width", type=int, default=3840)
    ap.add_argument("--height", type=int, default=2160)
    ap.add_argument("--seed", type=int, default=1)
    ap.add_argument("--intra-pct", type=int, default=15)
    ap.add_argument("--isp-pct", type=int, default=20)
    ap.add_argument("--distinct", type=int, default=6)


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    add_args(ap)
    ap.add_argument("--b-pictures", type=int, default=6, help="B pictures of the schedule to analyse")
    args = ap.parse_args()
    _, pics = bench_pictures(args)
    print(f"{'picture':8} {'blocks':>8} {'roots':>8} {'depth':>7} {'median samples':>15}")
    for name, pic in pics:
        d = depth(pic.get("intraTus", np.zeros(0, abi.INTRA_TU_DTYPE)), args.width, args.height)
        print(f"{name:8} {d['blocks']:8d} {d['roots']:8d} {d['depth']:7d} {d['median_samples']:15d}", flush=True)
