"""Diagnosis of a stream that decodes differently through the swapped decoder (test infrastructure): for a seed of tools/stream_fuzz.py (optionally with
overridden configuration entries, e.g. deblocking_disabled=True sao=False to take the in-loop filters out), prints for the first picture that differs a map of the
differing 8x8 blocks per plane and the flattened PU / TU / intra records that cover the first differing sample (stream_util.describe_difference).
    python tools/stream_diag.py SEED [key=value ...]"""
import sys, numpy as np
import os
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__))); sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tools"))
from oracle import vvc_stream as vs
from tests import helpers, stream_util as su
import stream_fuzz as sf
oracle = helpers.load_oracle()
seed = int(sys.argv[1])
kw, pics, st = sf.random_case(seed)
for a in sys.argv[2:]:
    k, v = a.split("="); kw[k] = eval(v)
aus, drawn, nb = vs.build_stream(vs.Config(**kw), pics, seed=seed)
keep = []
stock = vs.decode(vs.REF_SO, aus); sw, log = su.decode_swapped_cpu(aus, oracle, keep=keep)
frame = vs.output_order(pics)                                       # decoding index -> output index
np.set_printoptions(linewidth=250)
for i, rec in sorted(enumerate(keep), key=lambda e: frame[e[0]]):
    a, b = sw[frame[i]], stock[frame[i]]
    if all((x == y).all() for x, y in zip(a, b)): continue
    pic = rec["pic"]
    print("poc", rec["poc"], "slice types", pics[i].slice_type, pics[i].slice_types)
    for c in range(3):
        d = (a[c] != b[c])
        if not d.any(): continue
        B = 8 if c == 0 else 4
        H, W = d.shape; g = d[:H // B * B, :W // B * B].reshape(H // B, B, W // B, B).any(axis=(1, 3))
        print("plane", c, "blocks (8x8 luma units) with diffs:")
        for r in range(g.shape[0]):
            if g[r].any(): print("%3d " % (r * 8), "".join("#" if v else "." for v in g[r]))
    print(su.describe_difference(pic, a, b, 3 if rec["geom"].chromaFormat else 1))
    print("alf ctus", pic["alf"]["ctus"] if "alf" in pic else None)
    print("sao", pic.get("sao"))
    break
