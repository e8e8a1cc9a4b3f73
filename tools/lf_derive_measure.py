"""What the device edge derivation (B200_PIC_DERIVE_LF) changes for the bench's 4K pictures: host-to-device bytes per picture, the host CPU time of the
drop-in class's boundary-strength stage (DecLibReconB200 m_cpuNs[1]: calcFilterStrengthsCTU + flattenLfCtu without the derivation, the CU / TU record walk with
it), and — with --device, on the GPU — the device time of the new kernel family next to K3's.

    python tools/lf_derive_measure.py [--width 3840 --height 2160] [--pictures 4] [--threads 16] [--device] [--out FILE.json]

The pictures are bench.py's workload (same generator, seed and tool mix): its I picture and the first B pictures of its schedule.  The byte counts are computed
from the work lists; the host times are CPU time summed over the pool's threads (dry runs, no device); the device times are CUDA events around each kernel
family (b200_ctx_get_kernel_ms_n) over resident replays of one uploaded picture, after warm-up replays."""
import argparse, ctypes as C, json, os, sys, tempfile
import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from tests import helpers                                                     # noqa: E402
from vvdec_b200 import abi                                                    # noqa: E402


def flatten(ref, case, derive, threads):
    """One dry run of the drop-in class: (picture struct, Bs-stage CPU ms)."""
    os.environ["B200_LF_DERIVE"] = "1" if derive else "0"; os.environ["SEAM_TIMING"] = "1"
    h = case.build(); flat = abi.Picture(); col = np.zeros(ref.ref_seam_col_motion_bytes(h), np.uint8)
    with tempfile.TemporaryFile() as err:
        sys.stderr.flush(); saved = os.dup(2); os.dup2(err.fileno(), 2)
        try: secs = ref.ref_seam_run_b200(h, threads, 1, None, col.ctypes.data, len(col), C.byref(flat))
        finally: os.dup2(saved, 2); os.close(saved)
        err.seek(0); text = err.read().decode(errors="replace")
    ref.ref_seam_destroy(h)
    del os.environ["SEAM_TIMING"]; del os.environ["B200_LF_DERIVE"]
    assert secs >= 0, f"the drop-in class refused the picture ({secs})"
    line = [l for l in text.splitlines() if "Bs + grid" in l][-1]
    return flat, float(line.split("Bs + grid")[1].split("|")[0])


def h2d_bytes(flat, g, derive):
    """Bytes b200_pic_upload copies for the picture: the work lists, and either the two edge grids or the CU / TU records."""
    nCtu = ((g.width + g.ctuSize - 1) // g.ctuSize) * ((g.height + g.ctuSize - 1) // g.ctuSize)
    n4 = (g.width >> 2) * (g.height >> 2)
    common = 64 * flat.numPus + 32 * flat.numTus + 2 * flat.numCoefs + 4 * flat.numScaling + 16 * flat.numIntraTus + 24 * flat.numWp
    common += (nCtu if flat.ctuSlice else 0) + (24 * nCtu if flat.flags & abi.PIC_SAO else 0) + (8 * nCtu if flat.flags & abi.PIC_ALF else 0)
    lf = 24 * flat.numLfCus + 16 * flat.numLfTus + 4 * (nCtu + 1) + flat.numLfSlices if derive else 2 * 6 * n4
    return common + lf, lf


def device_times(lib, case, flat, reps):
    """ms per picture of every kernel family over `reps` resident replays of the derived picture (B200_PIC_DERIVE_LF)."""
    import vvdec_b200
    g = case.g
    pic = helpers.picture_from_struct(flat, g, case.filt)
    nCtu = ((g.width + g.ctuSize - 1) // g.ctuSize) * ((g.height + g.ctuSize - 1) // g.ctuSize)
    cp = lambda p, n, dt: np.frombuffer((C.c_uint8 * (n * np.dtype(dt).itemsize)).from_address(p), dt).copy()
    keep = dict(cus=cp(flat.lfCus, flat.numLfCus, abi.LF_CU_DTYPE), tus=cp(flat.lfTus, flat.numLfTus, abi.LF_TU_DTYPE),
                ctu=cp(flat.lfCtuCus, nCtu + 1, np.uint32), sb=cp(flat.lfSliceB, flat.numLfSlices, np.uint8))
    p = pic["struct"]
    p.flags |= abi.PIC_DERIVE_LF; p.lfV = p.lfH = None
    p.lfCus, p.numLfCus, p.lfTus, p.numLfTus = keep["cus"].ctypes.data, len(keep["cus"]), keep["tus"].ctypes.data, len(keep["tus"])
    p.lfCtuCus, p.lfSliceB = keep["ctu"].ctypes.data, keep["sb"].ctypes.data
    ctx = C.c_void_p()
    vvdec_b200.check(lib.b200_ctx_create(C.byref(ctx), C.byref(g), 17, 2, 0))
    try:
        for s in range(len(case.refs)): vvdec_b200.check(lib.b200_ctx_load_slot(ctx, s, abi.plane_ptrs(case.refs[s])))
        h = lib.b200_pic_upload(ctx, C.byref(p)); assert h >= 0, lib.b200_last_error()
        for _ in range(5): vvdec_b200.check(lib.b200_pic_run(ctx, h))            # warm-up
        vvdec_b200.check(lib.b200_wait_picture(ctx, h, None, 0))
        n = 11  # B200_KF_COUNT
        ms, cnt = (C.c_float * n)(), (C.c_int * n)()
        vvdec_b200.check(lib.b200_ctx_get_kernel_ms_n(ctx, ms, cnt, n))         # drop the warm-up
        vvdec_b200.check(lib.b200_ctx_set_profiling(ctx, 1))
        for _ in range(reps): vvdec_b200.check(lib.b200_pic_run(ctx, h))
        vvdec_b200.check(lib.b200_wait_picture(ctx, h, None, 0))
        vvdec_b200.check(lib.b200_ctx_get_kernel_ms_n(ctx, ms, cnt, n))
    finally:
        lib.b200_ctx_destroy(ctx)
    names = ["mc_tile", "mc_affine", "k1", "lf_v", "lf_h", "sao", "alf_luma", "alf_chroma", "intra", "lmcs", "lf_derive"]
    return {names[i]: round(ms[i] / reps, 4) for i in range(n) if cnt[i]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--width", type=int, default=3840); ap.add_argument("--height", type=int, default=2160)
    ap.add_argument("--pictures", type=int, default=4, help="the I picture and the first pictures-1 B pictures of bench.py's schedule")
    ap.add_argument("--threads", type=int, default=16); ap.add_argument("--repeat", type=int, default=3, help="host runs per picture and mode (median)")
    ap.add_argument("--device", action="store_true"); ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--seed", type=int, default=1); ap.add_argument("--intra-pct", type=int, default=15); ap.add_argument("--isp-pct", type=int, default=20)
    ap.add_argument("--out")
    a = ap.parse_args()
    ref = helpers.load_ref()
    rng = np.random.default_rng(a.seed)                                      # as bench.py's Workload (rank 0)
    base = helpers.SeamCase(ref, rng, a.width, a.height, intra=a.intra_pct, isp=a.isp_pct)
    seeds = [int(s) for s in rng.integers(1, 1 << 30, size=6 + 1)]
    cases = [("I", base.variant(seeds[-1], slice_type=2))] + [(f"B{k}", base.variant(seeds[k])) for k in range(a.pictures - 1)]
    out = {"geometry": f"{a.width}x{a.height}", "threads": a.threads, "pictures": []}
    lib = None
    if a.device:
        import vvdec_b200
        lib = vvdec_b200.lib()
        out["gpu"] = os.popen("nvidia-smi --query-gpu=name,power.limit --format=csv,noheader").read().strip()
    for name, case in cases:
        row = {"picture": name}
        for derive in (False, True):
            t = []
            for _ in range(a.repeat):
                flat, ms = flatten(ref, case, derive, a.threads); t.append(ms)
            total, lf = h2d_bytes(flat, case.g, derive)
            key = "derive" if derive else "grids"
            row[key] = {"h2d_bytes": total, "h2d_lf_bytes": lf, "bs_stage_cpu_ms": round(float(np.median(t)), 3)}
            if derive: row["cus"], row["tus"] = int(flat.numLfCus), int(flat.numLfTus)
            if derive and lib is not None: row["device_ms"] = device_times(lib, case, flat, a.reps)
        out["pictures"].append(row)
        print(json.dumps(row), flush=True)
    if a.out:
        with open(a.out, "w") as f: json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
