#!/usr/bin/env python
"""Clock trace of nms_peaks_persist_kernel on the bench workload (development aid).  Needs the trace build
(`make -C improved_body_parts_b200/csrc trace`, or another trace build named by SPG_LIB).  Runs the peak stage alone
after a warm-up pass and splits, per traced CTA (the first 64) and plane, the plane slot's cycle into its parts:

  copy      copy issued -> first scanner past `full` (the plane landed and a scanner was free to look at it)
  scan      first scanner past `full` -> last scanner done with the plane, less `wlist`
  wlist     the scanners waiting for a free peak list: last past `lfree` - last out of pass 1
  finish    last scanner done -> the finisher releases the slot (it refines from the staged plane)
  empty     the slot released -> the loader issues the slot's next copy (the slot stands empty)

and reports per plane: the scanners' spread (first -> last done), pass 1 (first past `full` -> last out of pass 1),
the loader's wait on `free`, the finisher's time (start -> end) and its wait for the list, peaks and queued groups.

usage: python tools/trace_nms_peaks.py [persons] [out.json]"""
import ctypes as C, json, os, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np, torch
from improved_body_parts_b200 import grouping, skeleton, synth

grouping.LIB_PATH = os.environ.get("SPG_LIB") or os.path.join(ROOT, "improved_body_parts_b200", "libspgroup_trace.so")
P = int(sys.argv[1]) if len(sys.argv) > 1 else 30
OUT = sys.argv[2] if len(sys.argv) > 2 else None
NB, CTAS, SLOTS, W, RING = 256, 64, 1024, 16, 3   # W, RING: kNmsTrWords, kNmsPSlots
heat, paf = synth.make_batch(20260921, NB, 128, 128, P)
dev = torch.device("cuda:0")
hd, pd = torch.from_numpy(heat).to(dev), torch.from_numpy(paf).to(dev)
prm = skeleton.default_params()
g = grouping.Grouper(max_batch=NB, max_person_rows=64)
lib = grouping.load_library()
lib.spg_trace_read.argtypes = [C.c_void_p, C.c_size_t, C.c_int]
buf = np.zeros(CTAS * SLOTS, dtype=np.uint64)
for _ in range(3):
    g.group_device(hd, pd, 128, prm)
torch.cuda.synchronize()
assert lib.spg_trace_read(buf.ctypes.data, buf.size, 1) == 0
g.nms_peaks(hd, prm)
torch.cuda.synchronize()
assert g.stage_kernels()[0] == "nms_peaks_persist_kernel", g.stage_kernels()
assert lib.spg_trace_read(buf.ctypes.data, buf.size, 1) == 0
tr = buf.reshape(CTAS, SLOTS // W, W).astype(np.int64)

rows = []
for b in range(CTAS):
    t = tr[b]
    nj = int(np.count_nonzero(t[:, 1]))
    t0 = int(t[0, 1])
    for j in range(nj):
        x = t[j]
        nxt = int(tr[b, j + RING, 1]) if j + RING < nj else 0
        wlist = max(int(x[4] - x[5]), 0)
        rows.append({"cta": b, "j": j, "issue": int(x[1] - t0), "full": int(x[2] - t0), "freed": int(x[10] - t0),
                     "copy": int(x[2] - x[1]), "scan": int(x[7] - x[2]) - wlist, "wlist": wlist,
                     "finish": int(x[10] - x[7]), "empty": nxt - int(x[10]) if nxt else None, "cycle": nxt - int(x[1]) if nxt else None,
                     "spread": int(x[7] - x[6]), "pass1": int(x[5] - x[2]), "loader_wait": int(x[1] - x[0]),
                     "fin": int(x[10] - x[9]), "fin_wait": int(x[9] - x[13]), "ready_to_fin": int(x[9] - x[8]),
                     "peaks": int(x[12]), "queued": int(x[11])})
if OUT:
    json.dump(rows, open(OUT, "w"))
# steady state only: the first 2 * RING planes of a CTA fill the plane ring and the list ring, the last RING have no successor
st = [r for r in rows if r["j"] >= 2 * RING and r["cycle"] is not None]
mean = lambda k: float(np.mean([r[k] for r in st if r[k] is not None]))
span = np.mean([max(r["freed"] for r in rows if r["cta"] == b) for b in range(CTAS)])
print(f"persons {P}: {len(st)} steady-state planes over {CTAS} CTAs, CTA span (first issue -> last free) {span:.0f} cycles")
print("cycles per plane slot (mean): cycle %.0f = copy %.0f + scan %.0f + wait-for-list %.0f + finish %.0f + empty %.0f" % (
    mean("cycle"), mean("copy"), mean("scan"), mean("wlist"), mean("finish"), mean("empty")))
print("  scanners: pass 1 %.0f, spread first->last done %.0f; loader wait on free %.0f" % (
    mean("pass1"), mean("spread"), mean("loader_wait")))
print("  finisher: %.0f per plane, waited %.0f for the list, started %.0f after it was ready" % (
    mean("fin"), mean("fin_wait"), mean("ready_to_fin")))
print("  peaks per plane %.1f, queued groups per plane %.1f" % (mean("peaks"), mean("queued")))
