"""Timeline of CTA 0 of the transposed kernel (diagnostic build: make -C nyx_b200/csrc EXTRA=-DNYXB_TX_TRACE, run with
NYXB_TX_TRACE_FILE=out.bin): python scripts/tx_trace.py out.bin [walkers=8] [helpers per set=2]
Prints, in SM clocks: walk duration (all walkers and per scheduler), walker wait per walk, helper latency DONE -> READY (post),
READY -> next DONE wait (slack), the serial stretch between two attempts, and how long a published stage waits for the walkers.
Helper 0 of a set is the lead (position side, DCMs, controller); helper 1 reduces the partial sums and assembles the accelerations."""
import sys
import numpy as np

CAP = 8192
NAMES = {1: "POLL", 2: "WALK", 3: "WALK_END", 4: "DONE_WAIT", 5: "DONE_SEEN", 6: "READY", 7: "STAGES_END", 8: "CTRL_END", 9: "TOP", 10: "PRE_DONE", 11: "DCM_DONE", 12: "REDUCED", 13: "ACC_DONE", 14: "HB_PASSED"}
raw = np.fromfile(sys.argv[1], dtype=np.uint64).reshape(32, CAP)
P = int(sys.argv[2]) if len(sys.argv) > 2 else 8
HW = int(sys.argv[3]) if len(sys.argv) > 3 else 2


def decode(strip):
    strip = strip[strip != 0]
    return (strip >> np.uint64(20)).astype(np.int64), ((strip >> np.uint64(12)) & np.uint64(0xff)).astype(int), \
        ((strip >> np.uint64(8)) & np.uint64(0xf)).astype(int), (strip & np.uint64(0xff)).astype(int)


def stats(name, x):
    x = np.asarray(x, dtype=float)
    if len(x) == 0:
        print(f"  {name:46s} (none)"); return
    print(f"  {name:46s} n={len(x):6d}  mean {x.mean():8.0f}  p10 {np.percentile(x,10):7.0f}  median {np.median(x):7.0f}  p90 {np.percentile(x,90):7.0f}  max {x.max():8.0f}")


t0 = min(decode(raw[w])[0][0] for w in range(32) if (raw[w] != 0).any())
walk_end = {}    # (ctx, walk ordinal of that ctx) -> latest WALK_END over the walkers
walk_start = {}
print("walkers:")
allw, allp = [], []
per_sched = {}
for w in range(P):
    t, code, ctx, stg = decode(raw[w])
    ordn = {0: 0, 1: 0}
    i = 0
    while i + 2 < len(t):
        if code[i] == 1 and code[i + 1] == 2 and code[i + 2] == 3:
            c = ctx[i + 1]
            allp.append(t[i + 1] - t[i]); allw.append(t[i + 2] - t[i + 1])
            per_sched.setdefault(w % 4, []).append(t[i + 2] - t[i + 1])
            k = (c, ordn[c]); ordn[c] += 1
            walk_end[k] = max(walk_end.get(k, 0), t[i + 2]); walk_start[k] = min(walk_start.get(k, 1 << 62), t[i + 1])
            i += 3
        else:
            i += 1
stats("walk (READY seen -> DONE arrive)", allw)
for sc in sorted(per_sched):
    stats(f"walk on scheduler {sc} (walkers {', '.join(str(w) for w in range(P) if w % 4 == sc)})", per_sched[sc])
stats("wait before a walk (poll)", allp)
print(f"  walkers busy {100 * sum(allw) / (sum(allw) + sum(allp)):.1f} % of their time")
print("helpers (lead = first helper of a context):")
for h in range(P, P + 2 * HW):
    t, code, ctx, stg = decode(raw[h])
    if len(t) == 0: continue
    c = (h - P) // HW
    post, slack, dwait, ready_at = [], [], [], {}
    last_ready = None
    ordn = 0
    for i in range(len(t) - 1):
        if code[i] == 4 and code[i + 1] == 5:
            dwait.append(t[i + 1] - t[i])
            if last_ready is not None: slack.append(t[i] - last_ready)
        if code[i] == 5:
            j = i + 1
            while j < len(t) and code[j] not in (6, 7, 4): j += 1
            if j < len(t) and code[j] == 6: post.append(t[j] - t[i])
        if code[i] == 6: last_ready = t[i]
    bound = [t[j] - t[i] for i in range(len(t)) if code[i] == 7 for j in range(i + 1, min(i + 6, len(t))) if code[j] == 6 and stg[j] == 0][:10000]
    print(f" helper warp {h} (context {c}, helper {(h - P) % HW}, scheduler {h % 4}):")
    seg = {}
    for i in range(len(t) - 1):
        if code[i] in (6, 10, 11, 5, 12, 13, 14) and code[i + 1] in (10, 11, 4, 12, 13, 14, 6) and stg[i] == stg[i + 1] or (code[i] == 6 and code[i + 1] == 10):
            seg.setdefault((NAMES[code[i]], NAMES[code[i + 1]]), []).append(t[i + 1] - t[i])
    for k in (("READY", "PRE_DONE"), ("PRE_DONE", "DCM_DONE"), ("DONE_SEEN", "REDUCED"), ("REDUCED", "ACC_DONE"), ("ACC_DONE", "HB_PASSED"), ("HB_PASSED", "READY")):
        if k in seg: stats("  " + k[0] + " -> " + k[1], seg[k])
    stats("wait for DONE", dwait); stats("post: DONE seen -> READY(i+2) published", post); stats("slack: READY published -> next DONE wait", slack)
    stats("between attempts: last stage done -> READY(0)", bound)
# how long does a published stage wait for the walkers? lead's READY(c, stage) vs first walker start of that walk
for c in range(2):
    t, code, ctx, stg = decode(raw[P + HW * c])
    ready = [t[i] for i in range(len(t)) if code[i] == 6]
    lat = [walk_start[(c, k)] - ready[k] for k in range(min(len(ready), sum(1 for kk in walk_start if kk[0] == c))) if (c, k) in walk_start]
    stats(f"context {c}: READY published -> first walker starts", lat)
    t5 = [t[i] for i in range(len(t)) if code[i] == 5]
    lat2 = [t5[k] - walk_end[(c, k)] for k in range(min(len(t5), sum(1 for kk in walk_end if kk[0] == c))) if (c, k) in walk_end]
    stats(f"context {c}: last walker done -> helper sees DONE", lat2)
