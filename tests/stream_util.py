"""Bitstream-level test plumbing: a stream written by oracle/vvc_stream.py decoded by (a) the stock reference and (b) the reference with the drop-in class behind
the DecLibRecon seam (oracle/_ref/libvvdec_swapped.so).  On a machine without a GPU (b) runs its host stages for real and the oracle chain in place of the device
(DecLibReconB200::TestHooks); on the GPU box it is the product path."""
import ctypes as C, numpy as np
from tests import helpers
from vvdec_b200 import abi
from oracle import vvc_stream as vs

NUM_SLOTS = 17                                                   # DecLibReconB200::m_dpbSlots

_HOOK = C.CFUNCTYPE(None, C.c_void_p, C.POINTER(abi.Picture), C.POINTER(abi.Geom), C.POINTER(C.c_int32), C.c_size_t,
                    C.POINTER(C.POINTER(C.c_int16)), C.POINTER(C.c_ssize_t), C.c_int)


_LOAD = C.CFUNCTYPE(None, C.c_void_p, C.c_int, C.POINTER(C.POINTER(C.c_int16)), C.POINTER(C.c_ssize_t), C.POINTER(abi.Geom))


def swapped_lib():
    lib = vs._lib(vs.SWAP_SO)
    lib.swapped_set_hooks.argtypes = [C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]
    lib.swapped_set_async_finish.argtypes = [C.c_int]
    return lib


class OracleDevice:
    """Stands where the device would: reconstructs every flattened picture with the oracle chain and keeps the decoded-picture buffer by slot."""
    def __init__(self, oracle):
        self.oracle, self.dpb, self.log, self.error = oracle, None, [], None
        self.keep, self.records = False, []                        # keep: a record of every picture handed over (replay, diagnosis; see _picture)
        self.cb = _HOOK(self._picture); self.load_cb = _LOAD(self._load)

    def _slots(self, g):
        if self.dpb is None or self.dpb[0][0].shape != (g.height, g.width):          # (first picture, or the context was rebuilt for another geometry)
            self.dpb = [[np.zeros((g.height, g.width), np.int16), np.zeros((g.height // 2, g.width // 2), np.int16), np.zeros((g.height // 2, g.width // 2), np.int16)]
                        for _ in range(NUM_SLOTS)]

    def _load(self, user, slot, planes, strides, geom):
        """b200_ctx_load_slot_strided: a reference the device does not hold is taken from its host planes"""
        try:
            g = geom.contents; self._slots(g)
            for c in range(3 if g.chromaFormat else 1):
                h, w = self.dpb[slot][c].shape
                src = np.ctypeslib.as_array(planes[c], shape=((h - 1) * strides[c] + w,))
                self.dpb[slot][c] = np.lib.stride_tricks.as_strided(src, shape=(h, w), strides=(strides[c] * 2, 2)).copy()
        except BaseException:
            import traceback; self.error = traceback.format_exc()

    def _picture(self, user, lists, geom, dmvr, ndmvr, planes, strides, poc):
        try:
            g = geom.contents; st = lists.contents
            self._slots(g)
            pic = helpers.picture_from_struct(st, g, None)
            if self.keep:                                             # the slots the PUs read, as they are before this picture is reconstructed
                refs = {int(s): [p.copy() for p in self.dpb[s]] for s in np.unique(pic["pus"]["refSlot"]) if s >= 0}
            out, dm = helpers.oracle_decompress(self.oracle, g, self.dpb, pic)
            self.dpb[st.dstSlot] = out
            if self.keep: self.records.append(dict(poc=int(poc), geom=abi.Geom.from_buffer_copy(g), pic=pic, refs=refs, out=out, dmvr=dm))
            n = min(int(ndmvr), len(dm))
            for i in range(n): dmvr[2 * i], dmvr[2 * i + 1] = int(dm[i][0]), int(dm[i][1])
            for c in range(3 if g.chromaFormat else 1):
                h, w = out[c].shape
                dst = np.ctypeslib.as_array(planes[c], shape=((h - 1) * strides[c] + w,))
                np.lib.stride_tricks.as_strided(dst, shape=(h, w), strides=(strides[c] * 2, 2))[...] = out[c]
            self.log.append(dict(poc=poc, slot=int(st.dstSlot), pus=int(st.numPus), tus=int(st.numTus), intra=int(st.numIntraTus), flags=int(st.flags), scaling=int(st.numScaling), wp=int(st.numWp), lfSlices=int(st.numLfSlices)))
        except BaseException as e:                                # never unwind through the C++ frames
            import traceback; self.error = traceback.format_exc()


def decode_swapped_cpu(aus, oracle, threads=1, keep=None, async_finish=False, **kw):
    """The stream through the swapped build without a device: glue host stages + oracle chain.  Returns (frames, per-picture log).
    keep: a list that receives one record per picture in the order the pictures are handed over: POC, geometry, flattened lists, the DPB slots its PUs
    reference, the oracle chain's planes and DMVR deltas."""
    lib = swapped_lib(); dev = OracleDevice(oracle)
    if keep is not None: dev.keep, dev.records = True, keep
    lib.swapped_set_hooks(1, C.cast(dev.cb, C.c_void_p), C.cast(dev.load_cb, C.c_void_p), None)
    lib.swapped_set_async_finish(int(async_finish))            # pictures complete in a pool task (DecLibReconB200::setAsyncFinish) instead of in waitForPrevDecompressedPic()
    try:
        frames = vs.decode(vs.SWAP_SO, aus, threads=threads, **kw)
    finally:
        lib.swapped_set_hooks(1, None, None, None); lib.swapped_set_async_finish(0)
    assert dev.error is None, dev.error
    return frames, dev.log


def decode_swapped_device(aus, threads=8, async_finish=False, **kw):
    """The stream through the swapped build on the product path (GPU)."""
    lib = swapped_lib(); lib.swapped_set_hooks(0, None, None, None); lib.swapped_set_async_finish(int(async_finish))
    try: return vs.decode(vs.SWAP_SO, aus, threads=threads, **kw)
    finally: lib.swapped_set_async_finish(0)


def corruption_run(seed, n, threads):
    """n streams with 1-3 flipped bits in a later access unit through the swapped build (oracle device); prints `ok` per stream that came back — with an error code
    or with frames — and exits.  Run in a child process (tests/test_stream_cpu.py): a crash or a hang of the class's error paths must not take the test run down."""
    import os
    from tests.test_stream_cpu import ALL, gop4, low_delay
    oracle = helpers.load_oracle(); rng = np.random.default_rng(seed)
    for it in range(n):
        aus, _, _ = vs.build_stream(vs.Config(**dict(ALL, sao=True)), low_delay(5) if it % 2 else gop4(), seed=int(rng.integers(1, 1 << 20)))
        k = int(rng.integers(1, len(aus))); au = bytearray(aus[k])
        for _ in range(int(rng.integers(1, 4))):
            au[int(rng.integers(12, len(au)))] ^= 1 << int(rng.integers(0, 8))
        bad = list(aus); bad[k] = bytes(au)
        try:
            frames, _ = decode_swapped_cpu(bad, oracle, threads=threads); print("ok frames", len(frames), flush=True)
        except vs.DecodeError as e:
            print("ok error", str(e).split("|")[0].strip(), flush=True)
    os._exit(0)


def device_child(in_path, out_path, threads, async_finish):
    """child process of decode_swapped_device_guarded(): decodes on the device path and stores the frames"""
    import os, pickle
    aus, kw = pickle.load(open(in_path, "rb"))
    try:
        frames = decode_swapped_device(aus, threads=threads, async_finish=async_finish, **kw)
        pickle.dump(dict(frames=frames, hash_errors=vs.decode.hash_errors), open(out_path, "wb"))
    except vs.DecodeError as e:
        pickle.dump(dict(error=str(e)), open(out_path, "wb"))
    os._exit(0)


def decode_swapped_device_guarded(aus, threads=4, async_finish=False, timeout=240, **kw):
    """decode_swapped_device() in a child process with a time limit: a crash or a hang on the device path fails the one test instead of taking the test run down.
    Returns (frames, hash errors)."""
    import os, pickle, subprocess, sys, tempfile
    with tempfile.TemporaryDirectory() as d:
        pickle.dump((aus, kw), open(os.path.join(d, "in.pkl"), "wb"))
        p = subprocess.run([sys.executable, "-m", "tests.stream_util", "device", os.path.join(d, "in.pkl"), os.path.join(d, "out.pkl"), str(threads), str(int(async_finish))],
                           capture_output=True, text=True, timeout=timeout, cwd=os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
        assert p.returncode == 0 and os.path.exists(os.path.join(d, "out.pkl")), f"device decode died (rc {p.returncode}): {p.stderr[-600:]}"
        r = pickle.load(open(os.path.join(d, "out.pkl"), "rb"))
    assert "error" not in r, r.get("error")
    return r["frames"], r["hash_errors"]


# ---- replay corpus: every picture of real parsed streams, as the glue hands it over, replayable on its own ----------------------------------------------
FUZZ_SEEDS = range(7000, 7200)


def _stream_fuzz():
    import os, sys
    tools = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tools")
    if tools not in sys.path: sys.path.insert(0, tools)
    import stream_fuzz
    return stream_fuzz


def corpus_names():
    """Every case of tests/test_stream_cpu.py at seeds 1 and 2, the stream with three geometries, and a fixed range of tools/stream_fuzz.py draws."""
    from tests.test_stream_cpu import CASES
    return [f"{n}-s{s}" for s in (1, 2) for n in CASES] + ["sequence_change"] + [f"fuzz{s}" for s in FUZZ_SEEDS]


def corpus_stream(name):
    """(access units, pictures in decoding order, frame_samples for vs.decode, whether the stream has tiles) of a corpus entry, seeded as the test or the
    tool it comes from seeds it"""
    from tests import test_stream_cpu as t
    if name == "sequence_change":
        aus, _ = t.sequence_change_stream()
        return aus, t.gop4() + t.gop4() + t.gop4(), 256 * 192 * 2, False
    if name.startswith("fuzz"):
        seed = int(name[4:]); kw, pics, _ = _stream_fuzz().random_case(seed)
        aus, _, _ = vs.build_stream(vs.Config(**kw), pics, seed=seed)
        return aus, pics, kw["width"] * kw["height"] * 2, bool(kw.get("tiles"))
    case, seed = name.rsplit("-s", 1); kw, make = t.CASES[case]; pics = make()
    aus, _, _ = vs.build_stream(vs.Config(**kw), pics, seed=int(seed) * 7 + len(case))
    return aus, pics, None, bool(kw.get("tiles"))


def capture(name, oracle):
    """The corpus stream `name` decoded by the stock build and by the swapped build with the oracle chain as the device.  Returns dict(name, records, stock,
    tiles): one record per picture in decoding order (see decode_swapped_cpu), each with `frame`, the index of its picture among the stock frames."""
    aus, pics, samples, tiles = corpus_stream(name)
    stock = vs.decode(vs.REF_SO, aus, frame_samples=samples)
    records = []
    decode_swapped_cpu(aus, oracle, keep=records, frame_samples=samples)
    order = vs.output_order(pics)
    assert len(records) == len(pics) == len(stock), (name, len(records), len(pics), len(stock))
    for i, r in enumerate(records):
        assert r["poc"] == pics[i].poc, (name, i, r["poc"], pics[i].poc)
        r["frame"] = order[i]
    return dict(name=name, records=records, stock=stock, tiles=tiles)


def sentinel_planes(g):
    """What every DPB slot holds before a replay loads the record's references: a wrong slot index reads this instead of the reference."""
    from vvdec_b200 import synth
    return synth.noise_planes(np.random.default_rng(g.width * 131 + g.height), g.width, g.height, g.bitDepth)


def oracle_replay(oracle, rec, flags=None):
    """The record's picture through the oracle chain from its snapshot alone (the other slots hold the sentinel).  flags: in place of the picture's
    b200_picture::flags.  Returns (planes, DMVR deltas)."""
    g, pic = rec["geom"], rec["pic"]; fill = sentinel_planes(g)
    dpb = [rec["refs"].get(s, fill) for s in range(NUM_SLOTS)]
    old = pic["struct"].flags
    if flags is not None: pic["struct"].flags = flags
    try: return helpers.oracle_decompress(oracle, g, dpb, pic)
    finally: pic["struct"].flags = old


def num_planes(g):
    return 3 if g.chromaFormat else 1


def first_difference(got, want, n):
    """(plane, number of differing samples, y, x, got sample, wanted sample) of the first plane among the first n that differs, or None"""
    for c in range(n):
        d = np.argwhere(got[c] != want[c])
        if len(d):
            y, x = (int(v) for v in d[0]); return c, len(d), y, x, int(got[c][y, x]), int(want[c][y, x])
    return None


def covering_records(pic, c, y, x):
    """The PU, TU and intra-block records of a picture's lists that cover sample (y, x) of plane c (chroma records on the chroma grid)."""
    X, Y = (x, y) if c == 0 else (2 * x, 2 * y)                       # luma position
    pus = pic["pus"]
    out = dict(pus=pus[(pus["x"] <= X) & (X < pus["x"] + pus["w"].astype(int)) & (pus["y"] <= Y) & (Y < pus["y"] + pus["h"].astype(int))])
    for key, recs in (("tus", pic["tus"]), ("intra", pic.get("intraTus"))):
        if recs is None: continue
        w = 1 << recs["log2w"].astype(int); h = 1 << recs["log2h"].astype(int); sc = np.where(recs["comp"] == 0, 1, 2)
        out[key] = recs[(recs["x"] * sc <= X) & (X < (recs["x"] + w) * sc) & (recs["y"] * sc <= Y) & (Y < (recs["y"] + h) * sc)]
    return out


def describe_difference(pic, got, want, n):
    """None when the first n planes agree; else the plane, the number of differing samples, the first one and the records that cover it"""
    d = first_difference(got, want, n)
    if d is None: return None
    c, k, y, x, a, b = d
    recs = covering_records(pic, c, y, x)
    return (f"plane {c}: {k} samples differ, first at (y={y}, x={x}): {a} vs {b}; covering records: "
            + "; ".join(f"{key} {v.dtype.names} {v.tolist()}" for key, v in recs.items()))


def pack(cap):
    """A capture() result as plain arrays and numbers (ctypes structs with pointers do not pickle): what a worker process sends back."""
    def pic_pack(pic):
        st = pic["struct"]
        d = {k: v for k, v in pic.items() if k not in ("struct", "alfTabs", "lmcs", "lfSeq")}
        d["meta"] = dict(dstSlot=st.dstSlot, flags=st.flags, numDmvr=st.numDmvr, numCoefs=st.numCoefs, numLfSlices=st.numLfSlices)
        if "alfTabs" in pic: T = pic["alfTabs"]; d["alfCounts"] = (T.numLumaSets, T.numChromaAlts, T.numCc[0], T.numCc[1])
        if "lmcs" in pic: d["lmcs"] = dict(raw=bytes(pic["lmcs"]["struct"]), invLUT=pic["lmcs"]["invLUT"], vpdus=pic["lmcs"]["vpdus"])
        if "lfSeq" in pic: d["lfSeq"] = bytes(pic["lfSeq"])
        return d
    recs = [dict(r, geom=bytes(r["geom"]), pic=pic_pack(r["pic"])) for r in cap["records"]]
    return dict(cap, records=recs)


def unpack(cap):
    """pack() undone: the records' lists as helpers.picture_from_struct makes them."""
    def pic_unpack(d, g):
        m = d["meta"]; p = abi.Picture(); keep = []
        p.dstSlot, p.flags, p.numDmvr = m["dstSlot"], m["flags"], m["numDmvr"]
        p.pus, p.numPus = d["pus"].ctypes.data, len(d["pus"]); p.tus, p.numTus = d["tus"].ctypes.data, len(d["tus"])
        p.coefs, p.numCoefs = d["coefs"].ctypes.data, m["numCoefs"]
        if "scaling" in d: p.scaling, p.numScaling = d["scaling"].ctypes.data, len(d["scaling"])
        if "intraTus" in d: p.intraTus, p.numIntraTus = d["intraTus"].ctypes.data, len(d["intraTus"])
        if m["flags"] & abi.PIC_DEBLOCK:
            p.lfV, p.lfH, p.lfSlices, p.numLfSlices = d["lfV"].ctypes.data, d["lfH"].ctypes.data, d["lfSlices"].ctypes.data, m["numLfSlices"]
            if "ctuSlice" in d: p.ctuSlice = d["ctuSlice"].ctypes.data
            if "lfSeq" in d: s = abi.LfSeq.from_buffer_copy(d["lfSeq"]); keep.append(s); p.lfSeq = C.addressof(s)
        if m["flags"] & abi.PIC_SAO: p.sao = d["sao"].ctypes.data
        if m["flags"] & abi.PIC_ALF:
            a = d["alfArrays"]; A = abi.AlfTables(); keep.append(A); p.alf = d["alf"]["ctus"].ctypes.data; p.alfTabs = C.addressof(A)
            A.lumaCoeff, A.lumaClip, A.chromaCoeff, A.chromaClip = (a[k].ctypes.data for k in ("lumaCoeff", "lumaClip", "chromaCoeff", "chromaClip"))
            A.ccCoeff[0], A.ccCoeff[1] = a["cc0"].ctypes.data, a["cc1"].ctypes.data
            A.numLumaSets, A.numChromaAlts, A.numCc[0], A.numCc[1] = d["alfCounts"]
        if "wp" in d: p.wp, p.numWp = d["wp"].ctypes.data, len(d["wp"])
        if m["flags"] & abi.PIC_LMCS:
            L = abi.Lmcs.from_buffer_copy(d["lmcs"]["raw"]); keep.append(L); p.lmcs = C.addressof(L)
            L.invLUT, L.vpdus = d["lmcs"]["invLUT"].ctypes.data, d["lmcs"]["vpdus"].ctypes.data
        return helpers.picture_from_struct(p, g, None)                  # (deep copies: nothing points into `d` or `keep` afterwards)
    recs = []
    for r in cap["records"]:
        g = abi.Geom.from_buffer_copy(r["geom"]); recs.append(dict(r, geom=g, pic=pic_unpack(r["pic"], g)))
    return dict(cap, records=recs)


_WORKER_ORACLE = None


def _worker_init():
    global _WORKER_ORACLE
    _WORKER_ORACLE = helpers.load_oracle()


def capture_packed(name):
    """capture() in a worker process (CapturePool), packed for the way back"""
    return pack(capture(name, _WORKER_ORACLE))


class CapturePool:
    """Runs fn(name) for the given corpus names in worker processes (spawned: the parent may hold a CUDA context), a bounded number ahead of the caller,
    and hands the results out in the order get() asks for them."""
    def __init__(self, names, fn, workers=None):
        import multiprocessing as mp, os
        self.names, self.fn, self.pending, self.next = list(names), fn, {}, 0
        n = max(1, min(len(self.names), workers or os.cpu_count() or 1, 16))
        self.pool, self.ahead = mp.get_context("spawn").Pool(n, initializer=_worker_init), 2 * n
        self._fill()

    def _fill(self):
        while self.next < len(self.names) and len(self.pending) < self.ahead:
            name = self.names[self.next]; self.next += 1
            self.pending[name] = self.pool.apply_async(self.fn, (name,))

    def get(self, name):
        r = (self.pending.pop(name) if name in self.pending else self.pool.apply_async(self.fn, (name,))).get(timeout=600)      # (a worker that died never answers)
        self._fill()
        return r

    def close(self):
        self.pool.terminate(); self.pool.join()


if __name__ == "__main__":
    import sys
    if sys.argv[1] == "device": device_child(sys.argv[2], sys.argv[3], int(sys.argv[4]), bool(int(sys.argv[5])))
    corruption_run(int(sys.argv[1]), int(sys.argv[2]), int(sys.argv[3]))
