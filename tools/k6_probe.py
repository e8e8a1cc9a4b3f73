"""Times the K6 launches of one I picture and one B picture of the bench workload (run under ncu for the per-kernel list)."""
import sys, os, ctypes as C, numpy as np
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__))); sys.path.insert(0, ROOT)
import vvdec_b200
from vvdec_b200 import abi
import bench
args = bench.parse()
lib = vvdec_b200.lib()
wl = bench.Workload(args, 0)
g = abi.make_geom(args.width, args.height, 10)
ctx = C.c_void_p(); vvdec_b200.check(lib.b200_ctx_create(C.byref(ctx), C.byref(g), 6, 2, 0))
for s in range(6): vvdec_b200.check(lib.b200_ctx_load_slot(ctx, s, abi.plane_ptrs(wl.base.refs[s % 4])))
for name, case in (("B", wl.B[0]), ("I", wl.I)):
    pic, _ = case.flatten(threads=os.cpu_count()); pic["struct"].dstSlot = 4
    h = lib.b200_pic_upload(ctx, C.byref(pic["struct"])); assert h >= 0
    for _ in range(3): vvdec_b200.check(lib.b200_pic_run(ctx, h))
    vvdec_b200.check(lib.b200_ctx_mark(ctx, 0))
    for _ in range(5): vvdec_b200.check(lib.b200_pic_run(ctx, h))
    vvdec_b200.check(lib.b200_ctx_mark(ctx, 1)); t = C.c_float(); vvdec_b200.check(lib.b200_ctx_elapsed_ms(ctx, C.byref(t)))
    print(name, "picture ms", t.value / 5, "intra blocks", len(pic.get("intraTus", [])), flush=True)
