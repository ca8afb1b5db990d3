#!/usr/bin/env python
"""Clock trace of limb_score_persist_kernel on the bench workload (development aid).  Needs the trace build
(`make -C improved_body_parts_b200/csrc trace`, or another trace build named by SPG_LIB).  Runs the scoring stage alone
after a warm-up pass and splits, per traced CTA (the first 64) and item, the plane slot's cycle into its parts:

  copy      copy issued -> first screener past `full` (plane landed and end-point lists published)
  screen    first screener past `full` -> last screener gone (the slot is free again)
  wait      last screener gone -> the loader issues the slot's next copy (the slot stands empty)
  exact     last screener gone -> last scorer gone (the meta slot, not the plane slot, is held)
  mfree     the loader waiting for a meta slot to come back from the scorers

It also times every CTA's start and exit with %globaltimer (one clock for all SMs) over SPAN_LAUNCHES launches and
prints the kernel span, the mean and the latest CTA exit and the mean exit per class blockIdx.x mod 6 (item = image * 30
+ limb: under a fixed grid stride of 132 CTAs, class c would only ever score the limbs k = c mod 6).

usage: python tools/trace_limb_score.py [persons] [out.json]"""
import ctypes as C, json, os, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np, torch
from improved_body_parts_b200 import grouping, skeleton, synth

grouping.LIB_PATH = os.environ.get("SPG_LIB") or os.path.join(ROOT, "improved_body_parts_b200", "libspgroup_trace.so")
P = int(sys.argv[1]) if len(sys.argv) > 1 else 30
OUT = sys.argv[2] if len(sys.argv) > 2 else None
NB, CTAS, SLOTS, W, RING = 256, 64, 1024, 16, 3   # W, RING: kTrItemWords, kPersistSlots
heat, paf = synth.make_batch(20260921, NB, 128, 128, P)
dev = torch.device("cuda:0")
hd, pd = torch.from_numpy(heat).to(dev), torch.from_numpy(paf).to(dev)
prm = skeleton.default_params()
g = grouping.Grouper(max_batch=NB, max_person_rows=64)
lib = grouping.load_library()
lib.spg_trace_read.argtypes = [C.c_void_p, C.c_size_t, C.c_int]
lib.spg_trace_read_spans.argtypes = [C.c_void_p, C.c_size_t, C.c_int]
SPAN_CTAS, SPAN_LAUNCHES, CLASSES = 1024, 20, 6   # kTraceSpanCtas
buf = np.zeros(CTAS * SLOTS, dtype=np.uint64)
spans = np.zeros(2 * SPAN_CTAS, dtype=np.uint64)
for _ in range(3):
    g.group_device(hd, pd, 128, prm)
torch.cuda.synchronize()
assert lib.spg_trace_read(buf.ctypes.data, buf.size, 1) == 0
assert lib.spg_trace_read_spans(spans.ctypes.data, spans.size, 1) == 0
assert "persist" in g.stage_kernels()[1]
exits, kspan = [], []   # per launch: CTA exits after the earliest CTA start (us), kernel span (us)
for i in range(SPAN_LAUNCHES):
    g.limb_score(pd, 128, prm)
    torch.cuda.synchronize()
    if i == 0:
        assert lib.spg_trace_read(buf.ctypes.data, buf.size, 1) == 0
    assert lib.spg_trace_read_spans(spans.ctypes.data, spans.size, 1) == 0
    s = spans.reshape(SPAN_CTAS, 2).astype(np.int64)
    s = s[: int(np.count_nonzero(s[:, 0]))]
    exits.append((s[:, 1] - s[:, 0].min()) / 1e3)
    kspan.append((s[:, 1].max() - s[:, 0].min()) / 1e3)
tr = buf.reshape(CTAS, SLOTS // W, W).astype(np.int64)

rows = []
for b in range(CTAS):
    t = tr[b]
    nj = int(np.count_nonzero(t[:, 8]))   # items closed (the end-of-queue header is published but never closed)
    t0 = int(t[0, 0])
    for j in range(nj):
        x = t[j]
        nxt = tr[b, j + RING, 1] if j + RING < nj else 0
        rows.append({"cta": b, "j": j, "issue": int(x[1] - t0), "full": int(x[5] - t0), "first_left": int(x[6] - t0),
                     "last_left": int(x[7] - t0), "exact_done": int(x[11] - t0) if x[11] else None,
                     "closed": int(x[8] - t0) if x[8] else None, "surv": int(x[9]), "cand": int(x[10]),
                     "copy": int(x[5] - x[1]), "screen": int(x[7] - x[5]), "screen_spread": int(x[7] - x[6]),
                     "wait": int(nxt - x[7]) if nxt else None, "cycle": int(nxt - x[1]) if nxt else None,
                     "exact": int(x[11] - x[7]) if x[11] else None,
                     "mfree": int(x[3] - x[2]) if x[3] else 0, "issue_stall": int(x[1] - x[0])})
if OUT:
    json.dump(rows, open(OUT, "w"))
# the first RING items of a CTA have no predecessor in their slot and the last RING no successor: steady state only
st = [r for r in rows if r["j"] >= RING and r["cycle"] is not None]
mean = lambda k: float(np.mean([r[k] for r in st if r[k] is not None]))
span = np.mean([max(r["closed"] or 0 for r in rows if r["cta"] == b) for b in range(CTAS)])
print(f"persons {P}: {len(st)} steady-state items over {CTAS} CTAs, CTA span {span:.0f} cycles")
print("cycles per item (mean): slot cycle %.0f = copy %.0f + screen %.0f + wait %.0f | screen spread (first->last warp) %.0f" % (
    mean("cycle"), mean("copy"), mean("screen"), mean("wait"), mean("screen_spread")))
print("  exact phase after the screen %.0f, loader stalled on mfree %.0f, loader stalled before the copy %.0f" % (
    mean("exact"), mean("mfree"), mean("issue_stall")))
print("  survivors per item %.1f, candidates per item %.1f" % (mean("surv"), mean("cand")))
ex = np.mean(exits, axis=0)   # per CTA, mean over the launches
cls = [float(np.mean(ex[c::CLASSES])) for c in range(CLASSES)]
print(f"CTA spans (%globaltimer, {len(ex)} CTAs, mean of {SPAN_LAUNCHES} launches, us): kernel span {np.mean(kspan):.1f}, "
      f"CTA exit mean {ex.mean():.1f} / latest {ex.max():.1f} / earliest {ex.min():.1f} "
      f"(latest - mean = {100 * (ex.max() - ex.mean()) / np.mean(kspan):.1f} % of the span)")
print("  mean exit per class blockIdx.x mod %d: %s" % (CLASSES, " / ".join(f"{c}: {v:.1f}" for c, v in enumerate(cls))))
