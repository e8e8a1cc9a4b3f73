"""The replay corpus on the device: every picture of real parsed streams (tests/stream_util.py corpus_names), replayed through b200_decompress_picture
from the records the glue handed over, bit-exact against the oracle chain's output recorded with them.

tests/test_stream_replay_cpu.py shows that each record replays through the oracle to the stock decoder's frame, so a difference here lies in a kernel or in
picture.cu.  Each picture with intra records runs under both K6 kernels; each replayed frame also goes through the output path (hashes, 8-bit and packed
10-bit frames, film grain) against the oracle on the stock frame.  Streams are captured in worker processes while the device replays earlier ones."""
import ctypes as C, os, numpy as np, pytest
import vvdec_b200
from oracle import vvc_stream as vs
from tests import helpers, stream_util as su
from vvdec_b200 import abi, synth

pytestmark = [pytest.mark.gpu, pytest.mark.skipif(not (vs.available() and os.path.exists(vs.SWAP_SO)), reason="oracle/_ref not built")]


@pytest.fixture(scope="module")
def captures(request):
    """the captures of the streams this run selected, in the order the tests ask for them"""
    names = [it.callspec.params["name"] for it in request.session.items if it.module is request.module and hasattr(it, "callspec")]
    pool = su.CapturePool(names, su.capture_packed)
    yield pool
    pool.close()


class Contexts:
    """One device context per geometry, with the glue's number of DPB slots, every slot filled with the sentinel picture when the context is made."""
    def __init__(self, b200):
        self.b200, self.ctxs = b200, {}

    def get(self, g):
        key = bytes(g)
        if key not in self.ctxs:
            if len(self.ctxs) >= 4: self.b200.b200_ctx_destroy(self.ctxs.pop(next(iter(self.ctxs))))
            ctx = C.c_void_p(); vvdec_b200.check(self.b200.b200_ctx_create(C.byref(ctx), C.byref(g), su.NUM_SLOTS, 2, -1))
            self.ctxs[key] = ctx
            fill = su.sentinel_planes(g)
            for s in range(su.NUM_SLOTS): vvdec_b200.check(self.b200.b200_ctx_load_slot(ctx, s, abi.plane_ptrs(fill)))
        return self.ctxs[key]

    def close(self):
        for ctx in self.ctxs.values(): self.b200.b200_ctx_destroy(ctx)


@pytest.fixture(scope="module")
def contexts(b200):
    ctxs = Contexts(b200)
    yield ctxs
    ctxs.close()


def run_device(b200, ctx, rec, kernel, flags=None):
    """The record's picture on the device: its reference slots loaded from the snapshot, b200_decompress_picture, b200_wait_picture with the DMVR buffer,
    b200_get_frame of the destination slot.  Returns (planes, DMVR deltas)."""
    g, pic = rec["geom"], rec["pic"]; st = pic["struct"]
    for s, planes in rec["refs"].items(): vvdec_b200.check(b200.b200_ctx_load_slot(ctx, s, abi.plane_ptrs(planes)))
    old = st.flags
    if flags is not None: st.flags = flags
    try:
        with helpers.intra_kernel(kernel): h = b200.b200_decompress_picture(ctx, C.byref(st))
    finally: st.flags = old
    assert h >= 0, b200.b200_last_error()
    dm = np.zeros((pic["ndmvr"] + 1, 2), np.int32)
    vvdec_b200.check(b200.b200_wait_picture(ctx, h, dm.ctypes.data, len(dm)))
    got = [np.zeros_like(p) for p in rec["out"]]
    vvdec_b200.check(b200.b200_get_frame(ctx, st.dstSlot, abi.plane_ptrs(got if g.chromaFormat else [got[0], None, None])))
    return got, dm


def first_stage_that_differs(b200, oracle, ctx, rec, kernel):
    """Re-runs the picture on both sides with ALF cleared from its flags, then SAO, then deblocking: the stage whose removal makes the difference go."""
    f, n = rec["pic"]["struct"].flags, su.num_planes(rec["geom"])
    for stage, clear in (("ALF", abi.PIC_ALF), ("SAO", abi.PIC_SAO), ("deblocking", abi.PIC_DEBLOCK)):
        if not f & clear: continue
        f &= ~clear
        got, _ = run_device(b200, ctx, rec, kernel, f); want, _ = su.oracle_replay(oracle, rec, f)
        if su.first_difference(got, want, n) is None: return stage
    return "reconstruction before the in-loop filters (K1 / K2 / K6 / LMCS)"


def make_grain(pattern, sLUT, pLUT, seeds, shift, present):
    fg = abi.FilmGrain()
    fg.pattern, fg.sLUT, fg.pLUT, fg.lineSeeds = pattern.ctypes.data, sLUT.ctypes.data, pLUT.ctypes.data, seeds.ctypes.data
    fg.scaleShift = shift
    for c in range(3): fg.compPresent[c] = int(present[c])
    return fg


def check_output_path(b200, oracle, ctx, g, slot, frame, what):
    """The output kernels on the replayed frame in `slot` against the oracle on the stock frame: CRC and checksum, the 8-bit frame, the packed 10-bit frame
    (pyuv), and film grain on frames wider than 128."""
    n, W, H, bd = su.num_planes(g), g.width, g.height, g.bitDepth
    planes = [np.ascontiguousarray(frame[c]) for c in range(n)]
    size = lambda c: (W, H) if c == 0 else (W >> 1, H >> 1)

    def wait(t):
        assert t >= 0, b200.b200_last_error()
        vvdec_b200.check(b200.b200_frame_wait(ctx, t))

    for method, k, label in ((1, 2, "CRC"), (2, 4, "checksum")):          # B200_HASH_CRC, B200_HASH_CHECKSUM: digest bytes per plane
        dig = np.full(12, 0xEE, np.uint8)
        wait(b200.b200_frame_hash_async(ctx, slot, method, dig.ctypes.data))
        for c in range(n):
            want = np.zeros(4, np.uint8)
            assert oracle.orc_plane_hash(method, bd, planes[c], planes[c].shape[1], *size(c), want) == k
            assert np.array_equal(dig[c * k:(c + 1) * k], want[:k]), f"{what}: {label} of plane {c}"

    def frame_bytes(fmt):
        outs = [np.zeros(max(1, b200.b200_frame_bytes(C.byref(g), fmt, c)), np.uint8) for c in range(3)]
        return outs, (C.c_void_p * 3)(*[o.ctypes.data if c < n else None for c, o in enumerate(outs)])

    for fmt in (2, 1) if bd == 10 else (2,):                            # B200_OUT_8, B200_OUT_PYUV
        outs, ptrs = frame_bytes(fmt)
        wait(b200.b200_get_frame_fmt_async(ctx, slot, fmt, ptrs))
        for c in range(n):
            want = np.zeros(len(outs[c]), np.uint8)
            if fmt == 1: oracle.orc_pack_pyuv(planes[c], planes[c].shape[1], *size(c), want)
            else: oracle.orc_narrow8(planes[c], planes[c].shape[1], *size(c), bd, want)
            assert np.array_equal(outs[c], want), f"{what}: {'pyuv' if fmt == 1 else '8-bit'} frame, plane {c}"
    if W > 128 and bd in (8, 10):
        rng = np.random.default_rng(W * 7 + H + slot)
        pattern, sLUT, pLUT, seeds = synth.gen_film_grain_tables(rng, H)
        shift = int(rng.integers(8, 14)) - (bd - 8); present = np.array((1, n > 1, n > 1), np.uint8)
        want = [p.copy() for p in planes] + [None] * (3 - n)
        strides = (C.c_ssize_t * 3)(*[p.shape[1] if p is not None else 0 for p in want])
        oracle.orc_film_grain(abi.plane_ptrs(want), strides, W, H, bd, pattern.ctypes.data, sLUT.ctypes.data, pLUT.ctypes.data, seeds.ctypes.data, shift, present.ctypes.data)
        outs, ptrs = frame_bytes(0)
        wait(b200.b200_get_frame_grain_async(ctx, slot, 0, ptrs, C.byref(make_grain(pattern, sLUT, pLUT, seeds, shift, present))))
        for c in range(n):
            w, h = size(c)
            assert np.array_equal(outs[c].view(np.int16).reshape(h, g.stride[c])[:, :w], want[c]), f"{what}: film grain, plane {c}"


@pytest.mark.parametrize("name", su.corpus_names())
def test_stream_replay_on_the_device(b200, oracle, captures, contexts, name):
    cap = su.unpack(captures.get(name))
    ctxs = contexts
    for rec in cap["records"]:
        g, pic = rec["geom"], rec["pic"]; ctx = ctxs.get(g); n = su.num_planes(g)
        it = pic.get("intraTus")
        kernels = ("v1", "v2") if it is not None else ("auto",)
        for kernel in kernels:
            got, dm = run_device(b200, ctx, rec, kernel)
            what = f"{name} POC {rec['poc']} ({g.width}x{g.height} CTU {g.ctuSize} {g.bitDepth} bit{' 4:0:0' if n == 1 else ''}, K6 {kernel})"
            why = su.describe_difference(pic, got, rec["out"], n)
            if why is not None:
                pytest.fail(f"{what}: {why}; first stage that differs: {first_stage_that_differs(b200, oracle, ctx, rec, kernel)}")
            assert np.array_equal(dm, rec["dmvr"]), f"{what}: DMVR deltas differ at entries {np.flatnonzero((dm != rec['dmvr']).any(axis=1))[:8].tolist()}"
        check_output_path(b200, oracle, ctx, g, pic["struct"].dstSlot, cap["stock"][rec["frame"]], f"{name} POC {rec['poc']}")
