"""Pictures in flight the way bench.py drives them, bit-exact against the oracle chain run serially on a host model of the DPB: uploads ahead of the
runs, resident handles replayed with no waits, asynchronous outputs of every kind while later pictures recycle the buffer they read, two contexts
on one device, and arenas / staging buffers that grow while pictures are in flight.  The schedules are tests/helpers.py:PIPELINE_SCHEDULES
(tests/test_pipeline_cases_cpu.py checks what they contain).

Host arrays whose copies should be asynchronous live in page-locked memory, each on pages of its own: a range that starts in a page registered for
another array makes copy2d_host fall back to a synchronous staged copy, and a copy to or from pageable memory is synchronous anyway; either would
hide the races these tests look for."""
import contextlib
import ctypes as C
import mmap
import numpy as np
import pytest
import vvdec_b200
from vvdec_b200 import abi, synth
from tests.helpers import oracle_decompress, pipeline_schedule, PIPELINE_SLOTS, intra_case

pytestmark = pytest.mark.gpu
PAGE = mmap.PAGESIZE
SLEEP_CYCLES = 100_000_000          # torch.cuda._sleep on the caller's side stream: ~50-70 ms on an H100, far longer than the pictures issued behind it
OUT_16, OUT_PYUV, OUT_8 = 0, 1, 2
HASH_CRC, HASH_CHECKSUM = 1, 2


class Pinned:
    """Page-locked host arrays, each registered on whole pages of its own (b200_host_register); unregistered by close()."""
    def __init__(self, b200):
        self.b200, self.regs, self.raw = b200, [], []

    def empty(self, shape, dtype):
        dtype = np.dtype(dtype)
        n = int(np.prod(shape)) * dtype.itemsize
        size = max(PAGE, -(-n // PAGE) * PAGE)
        raw = np.empty(size + PAGE, np.uint8)
        off = (-raw.ctypes.data) % PAGE
        vvdec_b200.check(self.b200.b200_host_register(raw.ctypes.data + off, size))
        self.regs.append(raw.ctypes.data + off); self.raw.append(raw)
        return raw[off:off + n].view(dtype).reshape(shape)

    def copy(self, a):
        out = self.empty(a.shape, a.dtype); out[...] = a
        return out

    def frame(self, W, H, dtype=np.int16):
        return [self.empty((H, W), dtype), self.empty((H // 2, W // 2), dtype), self.empty((H // 2, W // 2), dtype)]

    def close(self):
        for p in self.regs: self.b200.b200_host_unregister(p)
        self.regs = []


@contextlib.contextmanager
def pinned(b200):
    pool = Pinned(b200)
    try:
        yield pool
    finally:
        pool.close()


@contextlib.contextmanager
def context(b200, s, arenas):
    """A context on the schedule's geometry with its initial DPB loaded."""
    ctx = C.c_void_p()
    vvdec_b200.check(b200.b200_ctx_create(C.byref(ctx), C.byref(s["g"]), PIPELINE_SLOTS, arenas, -1))
    try:
        for k in range(PIPELINE_SLOTS): vvdec_b200.check(b200.b200_ctx_load_slot(ctx, k, abi.plane_ptrs(s["dpb"][k])))
        yield ctx
    finally:
        b200.b200_ctx_destroy(ctx)


def pin_picture(pool, pic, dst=None):
    """The picture's work lists copied into pinned arrays: (b200_picture pointing at them, the arrays, ctypes structs to keep alive)."""
    st = abi.Picture.from_buffer_copy(pic["struct"])
    if dst is not None: st.dstSlot = dst
    arrays, keep = [], []

    def pin(a):
        p = pool.copy(a); arrays.append(p)
        return p.ctypes.data
    st.pus, st.tus, st.coefs = pin(pic["pus"]), pin(pic["tus"]), pin(pic["coefs"])
    if "lfV" in pic: st.lfV, st.lfH, st.lfSlices = pin(pic["lfV"]), pin(pic["lfH"]), pin(pic["lfSlices"])
    if "sao" in pic: st.sao = pin(pic["sao"])
    if "alf" in pic:
        a = pic["alf"]; T = abi.AlfTables.from_buffer_copy(pic["alfTabs"]); keep.append(T)
        st.alf = pin(a["ctus"])
        T.lumaCoeff, T.lumaClip, T.chromaCoeff, T.chromaClip = pin(a["lumaCoeff"]), pin(a["lumaClip"]), pin(a["chromaCoeff"]), pin(a["chromaClip"])
        T.ccCoeff[0], T.ccCoeff[1] = pin(a["cc"][0]), pin(a["cc"][1])
        st.alfTabs = C.addressof(T)
    if "intraTus" in pic: st.intraTus = pin(pic["intraTus"])
    if "lmcs" in pic:
        L = abi.Lmcs.from_buffer_copy(pic["lmcs"]["struct"]); keep.append(L)
        L.invLUT, L.vpdus = pin(pic["lmcs"]["invLUT"]), pin(pic["lmcs"]["vpdus"])
        st.lmcs = C.addressof(L)
    keep.append(st)
    return st, arrays, keep


def scribble(arrays):
    for a in arrays: a.view(np.uint8).reshape(-1)[:] = 0xA5


_expected = {}


def expected(oracle, name, seq, dsts=None):
    """The oracle chain over the schedule's pictures seq[0], seq[1], ... (destination slots dsts, default the schedule's) on a host model of the DPB:
    per position (frame, DMVR deltas, destination slot), and the DPB after the last picture."""
    key = (name, tuple(seq), None if dsts is None else tuple(dsts))
    if key not in _expected:
        s = pipeline_schedule(name)
        dpb = [list(p) for p in s["dpb"]]
        out = []
        for j, k in enumerate(seq):
            dst = s["dsts"][k] if dsts is None else dsts[j]
            want, dm = oracle_decompress(oracle, s["g"], dpb, s["pics"][k])
            dpb[dst] = want
            out.append((want, dm, dst))
        _expected[key] = (out, dpb)
    return _expected[key]


def mismatch(what, got, want):
    for c, (a, b) in enumerate(zip(got, want)):
        a, b = np.asarray(a), np.asarray(b)
        if a.shape != b.shape: return f"{what}: plane {c}: shape {a.shape} vs {b.shape}"
        bad = np.argwhere(a != b)
        if len(bad):
            i = tuple(int(v) for v in bad[0])
            return f"{what}: plane {c}: {len(bad)} samples differ, first at {i}: {a[i]} vs {b[i]}"
    return None


def assert_same(what, got, want):
    msg = mismatch(what, got, want)
    assert msg is None, msg


def wait_dmvr(b200, ctx, handle, pic):
    dm = np.zeros((pic["ndmvr"] + 1, 2), np.int32)
    vvdec_b200.check(b200.b200_wait_picture(ctx, handle, dm.ctypes.data, len(dm)))
    return dm


# ---- a. upload ahead ----------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name,arenas", [("416x240", 1), ("416x240", 2), ("416x240", 3), ("416x240", 8), ("832x480", 3), ("1920x1080", 2)])
def test_upload_ahead(b200, oracle, name, arenas):
    """Up to arenas - 1 uploads ahead of the run (a parser running ahead of reconstruction), b200_pic_run with no waits, each frame read with
    b200_get_frame_async right after its run, the DMVR deltas read with b200_wait_picture just before the arena is uploaded again (as the glue does).
    The pinned work lists of a picture are overwritten as soon as b200_pic_run returns: it has waited for that picture's upload."""
    s = pipeline_schedule(name)
    n, W, H = len(s["pics"]), s["W"], s["H"]
    want, _ = expected(oracle, name, range(n))
    with pinned(b200) as pool, context(b200, s, arenas) as ctx:
        handles, lists, frames, tickets, dms = {}, {}, {}, [], {}
        for i in range(n):
            while len(handles) < min(n, i + arenas):
                k = len(handles)
                if k >= arenas: dms[k - arenas] = wait_dmvr(b200, ctx, handles[k - arenas], s["pics"][k - arenas])
                st, arrays, keep = pin_picture(pool, s["pics"][k])
                lists[k] = (arrays, keep)
                handles[k] = b200.b200_pic_upload(ctx, C.byref(st)); assert handles[k] == k % arenas, b200.b200_last_error()
            vvdec_b200.check(b200.b200_pic_run(ctx, handles[i]))
            scribble(lists[i][0])
            frames[i] = pool.frame(W, H)
            t = b200.b200_get_frame_async(ctx, s["dsts"][i], abi.plane_ptrs(frames[i])); assert t >= 0, b200.b200_last_error()
            tickets.append(t)
        for k in range(max(0, n - arenas), n): dms[k] = wait_dmvr(b200, ctx, handles[k], s["pics"][k])
        for t in tickets: vvdec_b200.check(b200.b200_frame_wait(ctx, t))
    for i in range(n):
        what = f"upload ahead {name} arenas {arenas}: step {i} ({s['kinds'][i]}) slot {s['dsts'][i]}"
        assert_same(what, frames[i], want[i][0])
        assert np.array_equal(dms[i], want[i][1]), f"{what}: DMVR deltas differ at {np.argwhere(dms[i] != want[i][1])[:3].tolist()}"


# ---- b. resident replay -------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", ["416x240", "832x480"])
def test_resident_replay(b200, oracle, name):
    """The bench's `value` leg: every distinct picture uploaded once, then the handles run in schedule order for two rounds with no waits, the I and
    LMCS handles twice back to back (a handle may be run several times; K6 resets its scratch on every launch).  Checkpoint frames are read
    asynchronously; each handle's DMVR deltas are those of its last run."""
    s = pipeline_schedule(name)
    n, W, H = len(s["pics"]), s["W"], s["H"]
    seq = []
    for _ in range(2):
        for k in range(n): seq += [k, k] if s["kinds"][k] in "IL" else [k]
    want, _ = expected(oracle, name, seq)
    with pinned(b200) as pool, context(b200, s, n) as ctx:
        keep = [pin_picture(pool, p) for p in s["pics"]]
        handles = [b200.b200_pic_upload(ctx, C.byref(st)) for st, _, _ in keep]
        assert handles == list(range(n)), b200.b200_last_error()
        vvdec_b200.check(b200.b200_wait_picture(ctx, -1, None, 0))
        frames, tickets = {}, []
        for j, k in enumerate(seq):
            vvdec_b200.check(b200.b200_pic_run(ctx, handles[k]))
            if j % 3 == 1 or j == len(seq) - 1:
                frames[j] = pool.frame(W, H)
                t = b200.b200_get_frame_async(ctx, s["dsts"][k], abi.plane_ptrs(frames[j])); assert t >= 0, b200.b200_last_error()
                tickets.append(t)
        dms = {k: wait_dmvr(b200, ctx, handles[k], s["pics"][k]) for k in range(n)}
        for t in tickets: vvdec_b200.check(b200.b200_frame_wait(ctx, t))
    for j, f in frames.items():
        assert_same(f"resident replay {name}: run {j} (picture {seq[j]}, {s['kinds'][seq[j]]}) slot {s['dsts'][seq[j]]}", f, want[j][0])
    for k in range(n):
        last = max(j for j, kk in enumerate(seq) if kk == k)
        assert np.array_equal(dms[k], want[last][1]), f"resident replay {name}: picture {k} DMVR deltas of run {last} differ"


# ---- c. asynchronous outputs while the buffer is recycled ---------------------------------------------------------------------------------
READERS = ("frame16", "fmt8", "pyuv", "crc", "checksum", "grain", "device")


class Readers:
    """Issues one output of each kind on a context and computes what it must hold from the expected frame."""
    def __init__(self, b200, oracle, pool, ctx, s, seed):
        import torch
        self.b200, self.oracle, self.pool, self.ctx, self.s, self.torch = b200, oracle, pool, ctx, s, torch
        self.side = torch.cuda.Stream()
        rng = np.random.default_rng(seed)
        tabs = synth.gen_film_grain_tables(rng, s["H"])
        self.grain = [pool.copy(t) for t in tabs]
        self.fg = abi.FilmGrain()
        self.fg.pattern, self.fg.sLUT, self.fg.pLUT, self.fg.lineSeeds = (t.ctypes.data for t in self.grain)
        self.fg.scaleShift = 9
        for c in range(3): self.fg.compPresent[c] = 1
        self.grain_want = [t.copy() for t in tabs]

    def issue(self, kind, slot, delay=False):
        """Returns a pending read: (kind, ticket or stream, destination)."""
        b, ctx, s = self.b200, self.ctx, self.s
        g, W, H = s["g"], s["W"], s["H"]
        if kind in ("frame16", "fmt8", "pyuv", "grain"):
            fmt = {"frame16": OUT_16, "fmt8": OUT_8, "pyuv": OUT_PYUV, "grain": OUT_16}[kind]
            dst = [self.pool.empty(b.b200_frame_bytes(C.byref(g), fmt, c), np.uint8) for c in range(3)]
            ptrs = (C.c_void_p * 3)(*[d.ctypes.data for d in dst])
            if kind == "frame16": t = b.b200_get_frame_async(ctx, slot, (C.POINTER(C.c_int16) * 3)(*[d.ctypes.data_as(C.POINTER(C.c_int16)) for d in dst]))
            elif kind == "grain": t = b.b200_get_frame_grain_async(ctx, slot, fmt, ptrs, C.byref(self.fg))
            else: t = b.b200_get_frame_fmt_async(ctx, slot, fmt, ptrs)
            assert t >= 0, b.b200_last_error()
            return kind, t, dst
        if kind in ("crc", "checksum"):
            dig = self.pool.empty(12, np.uint8); dig[:] = 0xEE
            t = b.b200_frame_hash_async(ctx, slot, HASH_CRC if kind == "crc" else HASH_CHECKSUM, dig.ctypes.data); assert t >= 0, b.b200_last_error()
            return kind, t, dig
        torch = self.torch
        dst = torch.full((W * H * 3 // 2,), -1, dtype=torch.int16, device="cuda")
        base = dst.data_ptr()
        pl = (C.c_void_p * 3)(base, base + 2 * W * H, base + 2 * (W * H + W * H // 4))
        self.side.wait_stream(torch.cuda.current_stream())                       # the fill of dst comes first
        if delay:
            with torch.cuda.stream(self.side): torch.cuda._sleep(SLEEP_CYCLES)
        vvdec_b200.check(b.b200_get_frame_device_async(ctx, slot, pl, C.c_void_p(self.side.cuda_stream)))
        return kind, self.side, dst

    def warm_up(self, handles, slot):
        """Runs the handles once and reads their slot in every way, then waits for all of it.  The first launch of a kernel may load its module, and
        that synchronises the device; the ordering tests then see only the waits the library itself asks for.  It also allocates the staging
        buffers, whose first growth drains the copy stream."""
        pending = []
        for h in handles:
            vvdec_b200.check(self.b200.b200_pic_run(self.ctx, h))
            pending += [self.issue(kind, slot) for kind in READERS]
        for p in pending: self.wait(p)
        vvdec_b200.check(self.b200.b200_wait_picture(self.ctx, -1, None, 0))

    def wait(self, pending):
        kind, t, dst = pending
        if kind == "device": t.synchronize()
        else: vvdec_b200.check(self.b200.b200_frame_wait(self.ctx, t))

    def got_want(self, pending, frame):
        """(what the read returned, what it must hold) as lists of arrays."""
        kind, _, dst = pending
        s, o = self.s, self.oracle
        W, H, bd = s["W"], s["H"], s["bd"]
        dims = [(W, H), (W // 2, H // 2), (W // 2, H // 2)]
        if kind == "device":
            flat = dst.cpu().numpy()
            return [flat[:W * H].reshape(H, W), flat[W * H:W * H * 5 // 4].reshape(H // 2, W // 2), flat[W * H * 5 // 4:].reshape(H // 2, W // 2)], frame
        if kind == "frame16": return [d.view(np.int16).reshape(f.shape) for d, f in zip(dst, frame)], frame
        if kind in ("fmt8", "pyuv"):
            want = [np.zeros(len(d), np.uint8) for d in dst]
            for c, (w, h) in enumerate(dims):
                if kind == "pyuv": o.orc_pack_pyuv(frame[c], frame[c].shape[1], w, h, want[c])
                else: o.orc_narrow8(frame[c], frame[c].shape[1], w, h, bd, want[c])
            return dst, want
        if kind in ("crc", "checksum"):
            m, nb = (HASH_CRC, 2) if kind == "crc" else (HASH_CHECKSUM, 4)
            want = []
            for c, (w, h) in enumerate(dims):
                d = np.zeros(4, np.uint8)
                assert o.orc_plane_hash(m, bd, frame[c], frame[c].shape[1], w, h, d) == nb
                want.append(d[:nb])
            return [dst[c * nb:(c + 1) * nb] for c in range(3)], want
        # grain, 16-bit output
        want = [f.copy() for f in frame]
        strides = (C.c_ssize_t * 3)(*[f.shape[1] for f in want])
        pat, sl, pl, seeds = self.grain_want
        pres = np.ones(3, np.uint8)
        o.orc_film_grain(abi.plane_ptrs(want), strides, W, H, bd, pat.ctypes.data, sl.ctypes.data, pl.ctypes.data, seeds.ctypes.data, self.fg.scaleShift, pres.ctypes.data)
        return [d.view(np.int16).reshape(f.shape) for d, f in zip(dst, frame)], want


@pytest.mark.parametrize("name", ["416x240", "832x480"])
def test_async_outputs_while_buffers_are_recycled(b200, oracle, name):
    """Every picture goes to slot 4, so the buffer a picture leaves in the slot is a work buffer of the picture after next.  Each picture's output is
    issued right after its run and waited for only after the next two pictures have been issued; the kinds rotate through every output path."""
    s = pipeline_schedule(name)
    n = len(s["pics"])
    seq = list(range(n)) * 2
    dsts = [4] * len(seq)
    want, _ = expected(oracle, name, seq, dsts)
    with pinned(b200) as pool, context(b200, s, 3) as ctx:
        rd = Readers(b200, oracle, pool, ctx, s, seed=n)
        keep = [pin_picture(pool, p, dst=4) for p in s["pics"]]
        pending, results = {}, {}
        for j, k in enumerate(seq):
            h = b200.b200_pic_upload(ctx, C.byref(keep[k][0])); assert h >= 0, b200.b200_last_error()
            vvdec_b200.check(b200.b200_pic_run(ctx, h))
            pending[j] = rd.issue(READERS[j % len(READERS)], 4)
            if j - 2 in pending:
                rd.wait(pending[j - 2]); results[j - 2] = rd.got_want(pending[j - 2], want[j - 2][0])
        for j in range(max(0, len(seq) - 2), len(seq)):
            rd.wait(pending[j]); results[j] = rd.got_want(pending[j], want[j][0])
    for j, (got, exp) in sorted(results.items()):
        assert_same(f"async outputs {name}: step {j} (picture {seq[j]}, {s['kinds'][seq[j]]}) slot 4, {READERS[j % len(READERS)]}", got, exp)


@pytest.mark.parametrize("case", ["alone", "second_reader", "load_slot"])
def test_delayed_device_reader(b200, oracle, case):
    """b200_get_frame_device_async on a side stream held back by a bounded sleep, so that its copy runs after later work has been issued.  alone: the
    next two pictures (the second recycles the buffer) must wait for it.  second_reader: a second reader of the same slot on the context's copy stream
    in between must not release the buffer before the first reader is done.  load_slot: b200_ctx_load_slot into that slot must wait for it too."""
    s = pipeline_schedule("416x240")
    seq, dsts = [0, 1, 2], [4, 4, 4]
    want, _ = expected(oracle, "416x240", seq, dsts)
    with pinned(b200) as pool, context(b200, s, 3) as ctx:
        rd = Readers(b200, oracle, pool, ctx, s, seed=7)
        keep = [pin_picture(pool, s["pics"][k], dst=4) for k in seq]
        hs = [b200.b200_pic_upload(ctx, C.byref(st)) for st, _, _ in keep]
        assert min(hs) >= 0, b200.b200_last_error()
        rd.warm_up(hs, 4)                               # slot 4 is no picture's reference: the runs below give the same frames
        vvdec_b200.check(b200.b200_pic_run(ctx, hs[0]))
        reads = [rd.issue("device", 4, delay=True)]
        if case == "second_reader": reads.append(rd.issue("frame16", 4))
        if case == "load_slot":
            other = s["dpb"][1]
            vvdec_b200.check(b200.b200_ctx_load_slot(ctx, 4, abi.plane_ptrs(other)))
        else:
            for h in hs[1:]: vvdec_b200.check(b200.b200_pic_run(ctx, h))
        for r in reads: rd.wait(r)
        results = [rd.got_want(r, want[0][0]) for r in reads]
        after = [np.zeros_like(p) for p in want[0][0]]
        vvdec_b200.check(b200.b200_get_frame(ctx, 4, abi.plane_ptrs(after)))
    for r, (got, exp) in zip(reads, results):
        assert_same(f"delayed reader ({case}): {r[0]} of step 0 slot 4", got, exp)
    assert_same(f"delayed reader ({case}): slot 4 afterwards", after, other if case == "load_slot" else want[2][0])


def test_grain_tables_are_copied_before_the_call_returns(b200, oracle):
    """b200_get_frame_grain_async promises that the tables are copied before it returns: pinned tables overwritten right after the call, while the copy
    stream is still held by an asynchronous read of the 1080p I picture, leave the grained frame as the original tables make it."""
    s = pipeline_schedule("1920x1080")
    want, _ = expected(oracle, "1920x1080", [0])
    with pinned(b200) as pool, context(b200, s, 1) as ctx:
        rd = Readers(b200, oracle, pool, ctx, s, seed=11)
        st, _, keep = pin_picture(pool, s["pics"][0])
        h = b200.b200_pic_upload(ctx, C.byref(st)); assert h == 0, b200.b200_last_error()
        rd.warm_up([h, h], 4)                           # twice: both grain staging buffers exist, so the call below drains nothing
        vvdec_b200.check(b200.b200_pic_run(ctx, h))
        first = rd.issue("frame16", 4)
        grained = rd.issue("grain", 4)
        rng = np.random.default_rng(12)
        for t, new in zip(rd.grain, synth.gen_film_grain_tables(rng, s["H"])): t[...] = new
        rd.wait(first); rd.wait(grained)
        results = [rd.got_want(first, want[0][0]), rd.got_want(grained, want[0][0])]
    for what, (got, exp) in zip(("frame16", "grain"), results):
        assert_same(f"grain tables: {what} of the I picture, slot 4", got, exp)


# ---- d. two contexts ----------------------------------------------------------------------------------------------------------------------
def test_two_contexts(b200, oracle):
    """Two lanes: two contexts on one device, each uploading one picture ahead, their b200_pic_run calls taking turns, asynchronous outputs on both,
    and a kernel-level call (b200_intra_reconstruct) in between.  Each context matches its own oracle run."""
    names = ("416x240", "832x480")
    sch = [pipeline_schedule(nm) for nm in names]
    wants = [expected(oracle, nm, range(len(s["pics"])))[0] for nm, s in zip(names, sch)]
    g6, planes6, resi6, recs6 = intra_case(W=256, H=128, ctu=32, min_size=4, p_isp=0.3, seed=21)
    want6 = [p.copy() for p in planes6]
    oracle.orc_intra_reconstruct(C.byref(g6), abi.plane_ptrs(want6), abi.plane_ptrs(resi6), recs6.ctypes.data, len(recs6))
    with pinned(b200) as pool, contextlib.ExitStack() as es:
        ctxs = [es.enter_context(context(b200, s, 2)) for s in sch]
        lists = [[pin_picture(pool, p) for p in s["pics"]] for s in sch]
        frames = [{}, {}]
        tickets = [[], []]
        nxt = [b200.b200_pic_upload(ctxs[l], C.byref(lists[l][0][0])) for l in range(2)]
        got6 = None
        for i in range(max(len(s["pics"]) for s in sch)):
            for l, s in enumerate(sch):
                if i >= len(s["pics"]): continue
                cur = nxt[l]; assert cur >= 0, b200.b200_last_error()
                if i + 1 < len(s["pics"]): nxt[l] = b200.b200_pic_upload(ctxs[l], C.byref(lists[l][i + 1][0]))
                vvdec_b200.check(b200.b200_pic_run(ctxs[l], cur))
                frames[l][i] = pool.frame(s["W"], s["H"])
                t = b200.b200_get_frame_async(ctxs[l], s["dsts"][i], abi.plane_ptrs(frames[l][i])); assert t >= 0, b200.b200_last_error()
                tickets[l].append(t)
            if i == 1:
                got6 = [p.copy() for p in planes6]
                vvdec_b200.check(b200.b200_intra_reconstruct(C.byref(g6), abi.plane_ptrs(got6), abi.plane_ptrs(resi6), recs6.ctypes.data, len(recs6)))
        for l in range(2):
            for t in tickets[l]: vvdec_b200.check(b200.b200_frame_wait(ctxs[l], t))
            vvdec_b200.check(b200.b200_wait_picture(ctxs[l], -1, None, 0))
    assert_same("two contexts: b200_intra_reconstruct in between", got6, want6)
    for l, s in enumerate(sch):
        for i, f in frames[l].items():
            assert_same(f"two contexts: lane {l} ({names[l]}) step {i} ({s['kinds'][i]}) slot {s['dsts'][i]}", f, wants[l][i][0])


# ---- e. growth and refusal while pictures are in flight -----------------------------------------------------------------------------------
def test_growth_while_in_flight(b200, oracle):
    """Small inter pictures, then larger lists uploaded into the arenas they held (b200_pic_upload reallocates) while earlier pictures run, the first
    intra picture arriving while inter-only pictures are in flight (the residual planes are allocated then), and the output format switching from
    8 bit to pyuv while earlier reads are pending (the staging buffers grow)."""
    name = "grow_416x240"
    s = pipeline_schedule(name)
    n = len(s["pics"])
    want, _ = expected(oracle, name, range(n))
    kinds = ("fmt8", "fmt8", "pyuv", "pyuv", "frame16")
    with pinned(b200) as pool, context(b200, s, 2) as ctx:
        rd = Readers(b200, oracle, pool, ctx, s, seed=5)
        lists = [pin_picture(pool, p) for p in s["pics"]]
        hs = [b200.b200_pic_upload(ctx, C.byref(lists[0][0]))]
        pending = []
        for i in range(n):
            if i + 1 < n: hs.append(b200.b200_pic_upload(ctx, C.byref(lists[i + 1][0])))
            assert hs[i] >= 0, b200.b200_last_error()
            vvdec_b200.check(b200.b200_pic_run(ctx, hs[i]))
            pending.append(rd.issue(kinds[i], s["dsts"][i]))
        for p in pending: rd.wait(p)
        results = [rd.got_want(p, want[i][0]) for i, p in enumerate(pending)]
        vvdec_b200.check(b200.b200_wait_picture(ctx, -1, None, 0))
    for i, (got, exp) in enumerate(results):
        assert_same(f"growth: step {i} ({s['kinds'][i]}) slot {s['dsts'][i]}, {kinds[i]}", got, exp)


def test_refused_picture_between_valid_ones(b200, oracle):
    """A picture with an invalid record, uploaded between valid pictures with uploads ahead, is refused by b200_pic_run; the slot mapping stays as it
    was, and the pictures after it are right."""
    name = "416x240"
    s = pipeline_schedule(name)
    n = len(s["pics"])
    want, dpb = expected(oracle, name, range(n))
    with pinned(b200) as pool, context(b200, s, 3) as ctx:
        lists = [pin_picture(pool, p) for p in s["pics"]]
        bad_st, bad_arrays, _ = pin_picture(pool, s["pics"][1], dst=s["dsts"][0])
        pus = bad_arrays[0].view(synth.PU_DTYPE)
        pus["refSlot"][3] = (17, -1)
        order = [("ok", 0), ("bad", None)] + [("ok", k) for k in range(1, n)]
        frames = {}
        queue = []
        for j, (what, k) in enumerate(order):
            st = bad_st if what == "bad" else lists[k][0]
            queue.append((what, k, b200.b200_pic_upload(ctx, C.byref(st))))
            if j >= 1:
                w, kk, h = queue.pop(0); assert h >= 0, b200.b200_last_error()
                rc = b200.b200_pic_run(ctx, h)
                if w == "bad":
                    assert rc == -2 and b"PU list" in b200.b200_last_error(), rc
                else:
                    vvdec_b200.check(rc)
                    frames[kk] = pool.frame(s["W"], s["H"])
                    vvdec_b200.check(b200.b200_frame_wait(ctx, b200.b200_get_frame_async(ctx, s["dsts"][kk], abi.plane_ptrs(frames[kk]))))
        for w, kk, h in queue:
            vvdec_b200.check(b200.b200_pic_run(ctx, h))
            frames[kk] = pool.frame(s["W"], s["H"])
            vvdec_b200.check(b200.b200_frame_wait(ctx, b200.b200_get_frame_async(ctx, s["dsts"][kk], abi.plane_ptrs(frames[kk]))))
        final = []
        for slot in range(PIPELINE_SLOTS):
            f = [np.zeros_like(p) for p in dpb[slot]]
            vvdec_b200.check(b200.b200_get_frame(ctx, slot, abi.plane_ptrs(f))); final.append(f)
    for k in range(n):
        assert_same(f"refusal: step {k} ({s['kinds'][k]}) slot {s['dsts'][k]}", frames[k], want[k][0])
    for slot in range(PIPELINE_SLOTS):
        assert_same(f"refusal: DPB slot {slot} at the end", final[slot], dpb[slot])
