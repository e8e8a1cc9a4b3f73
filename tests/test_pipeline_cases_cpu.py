"""The schedules of tests/test_pipeline_gpu.py reach what that file claims: the DPB slot patterns, both K6 kernels, the LMCS two-pass picture, CIIP
residuals, DMVR, filters on and off, and arenas that must grow while earlier pictures are in flight."""
import numpy as np
import pytest
from vvdec_b200 import abi
from tests.helpers import PIPELINE_SCHEDULES, pipeline_schedule, pipeline_refs, arena_bytes, intra_dense


@pytest.mark.parametrize("name", sorted(PIPELINE_SCHEDULES))
def test_pictures_are_what_their_kind_says(name):
    s = pipeline_schedule(name)
    g = s["g"]
    for i, (kind, pic) in enumerate(zip(s["kinds"], s["pics"])):
        it = pic.get("intraTus")
        n = 0 if it is None else len(it)
        st = pic["struct"]
        assert st.dstSlot == s["dsts"][i]
        if kind == "I":
            assert len(pic["pus"]) == 0 and intra_dense(g, n), (i, n)                        # the CTU-resident K6 kernel under auto
        elif kind in "BL":
            assert n and not intra_dense(g, n), (i, n)                                         # the one-CTA-per-block kernel
            ciip_resi = (it["ciip"] > 0) & ((it["flags"] & abi.INTRA_ADD_RESI) != 0) & ((it["flags"] & abi.INTRA_ISP) == 0)
            assert ciip_resi.any() and (it["ciip"] == 0).any(), i                               # the CIIP clear runs before K1; intra blocks too
            assert (pic["tus"]["flags"] & abi.TU_RESI).any()                                  # residual planes (resiBuf) in use
        else:
            assert n == 0 and len(pic["pus"])
        if kind == "L":
            assert st.flags & abi.PIC_LMCS and pic["lmcs"]["struct"].chromaAdj and (it["comp"] > 0).any() and (it["comp"] == 0).any()   # K6 in two passes
        else:
            assert not st.flags & abi.PIC_LMCS
        if kind == "P":
            assert pic["ndmvr"] > 0 and (pic["pus"]["flags"] & 2).sum() >= 10


@pytest.mark.parametrize("name", ["416x240", "832x480", "1920x1080"])
def test_slot_plans(name):
    """Each main schedule overwrites a slot the picture before it referenced, and has pictures whose result ends in each buffer the chain can leave
    it in: after ALF, after SAO without ALF, and in place (neither)."""
    s = pipeline_schedule(name)
    pics, dsts = s["pics"], s["dsts"]
    assert any(dsts[i + 1] in pipeline_refs(pics[i]) for i in range(len(pics) - 1))
    fl = [p["struct"].flags for p in pics]
    if name != "1920x1080":
        assert any(f & abi.PIC_ALF for f in fl) and any(f & abi.PIC_SAO and not f & abi.PIC_ALF for f in fl) and any(not f & (abi.PIC_SAO | abi.PIC_ALF) for f in fl)
        assert set("IBLP") <= set(s["kinds"])
    else:
        assert s["kinds"][0] == "I"                                                            # the long picture comes first
    if name == "416x240":
        assert any(dsts[i] == dsts[i + 1] for i in range(len(dsts) - 1))                       # a slot written twice in a row


def test_growing_arenas():
    """In the growth schedule, with two arenas, pictures 2 and 3 need more than the arenas pictures 0 and 1 left (DevBuf::reserve keeps a quarter
    more than it was asked for), so b200_pic_upload reallocates; picture 2 is the first with intra blocks (the residual planes are allocated then)."""
    s = pipeline_schedule("grow_416x240")
    g, pics = s["g"], s["pics"]
    sizes = [arena_bytes(g, p) for p in pics]
    cap = lambda n: n + (n >> 2) + 256
    assert sizes[2] > cap(sizes[0]) and sizes[3] > cap(sizes[1]), sizes
    assert all("intraTus" not in p for p in pics[:2]) and len(pics[2]["intraTus"])

