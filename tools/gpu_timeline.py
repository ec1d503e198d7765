#!/usr/bin/env python
"""Summarise a BWA_B200_GPUTRACE=1 log: how busy the GPU was between the first and the last timed stage, how much of that
time two or more lanes had a stage running, and where the idle gaps are.

    BWA_B200_GPUTRACE=1 python bench.py --worker ... 2> run.err;  python tools/gpu_timeline.py run.err [skip_ms]

Each `[gputrace] <lane> <stage:file:line> <t0> <t1>` line is one timed stage (kernel(s) or copy between two CUDA events of one lane's
stream), in ms on the device clock.  A stage's interval includes the time its kernels waited behind other streams' kernels, so
"sum of stages" exceeds wall time when lanes compete; "union" is the time at least one lane had a stage open."""
import collections
import re
import sys


def main():
    import gzip
    argv = [a for a in sys.argv[1:]]
    window = 0
    if "--window" in argv:
        k = argv.index("--window"); window = int(argv[k + 1]); del argv[k:k + 2]
    path = argv[0]
    skip = float(argv[1]) if len(argv) > 1 else 0.0
    iv = []
    for line in (gzip.open(path, "rt", errors="replace") if path.endswith(".gz") else open(path, errors="replace")):
        m = re.match(r"\[gputrace\] (\S+) (\S+) ([\d.]+) ([\d.]+)", line)
        if m:
            iv.append((float(m.group(3)), float(m.group(4)), m.group(1), m.group(2)))
    if not iv:
        print("no [gputrace] lines")
        return
    t_first = min(a for a, _, _, _ in iv)
    iv = [x for x in iv if x[0] >= t_first + skip]
    iv.sort()
    t0, t1 = iv[0][0], max(b for _, b, _, _ in iv)
    if window:
        k1 = [x for x in iv if x[3].startswith("smem:") or x[3] == "654"]   # (654: the seeding timer's line in older traces)
        if len(k1) >= window:
            best = min(range(len(k1) - window + 1), key=lambda s_: k1[s_ + window - 1][1] - k1[s_][0])
            t0, t1 = k1[best][0], k1[best + window - 1][1]
            iv = [(max(a, t0), min(b, t1), l, n) for a, b, l, n in iv if b > t0 and a < t1]
            print("window: %d seeding stages from the %dth, %.1f ms" % (window, best, t1 - t0))
    span = t1 - t0
    # union and overlap depth by sweeping the end points
    ev = sorted([(a, 1) for a, _, _, _ in iv] + [(b, -1) for _, b, _, _ in iv])
    depth, last, at_depth = 0, t0, collections.Counter()
    gaps = []
    for t, d in ev:
        at_depth[min(depth, 4)] += t - last
        if depth == 0 and t - last > 0:
            gaps.append((t - last, last))
        last = t
        depth += d
    print("stages %d, lanes %d, span %.1f ms" % (len(iv), len(set(x[2] for x in iv)), span))
    print("no stage open %.1f ms (%.1f%%), one %.1f%%, two %.1f%%, three %.1f%%, four or more %.1f%%" % (
        at_depth[0], 100 * at_depth[0] / span, 100 * at_depth[1] / span, 100 * at_depth[2] / span, 100 * at_depth[3] / span, 100 * at_depth[4] / span))
    by = collections.defaultdict(lambda: [0, 0.0])
    for a, b, _, ln in iv:
        by[ln][0] += 1
        by[ln][1] += b - a
    print("by stage (counter the timer adds to : the driver file and line of the timer): count, total ms, mean ms")
    for ln, (n, tot) in sorted(by.items(), key=lambda kv: -kv[1][1]):
        print("  %-16s %6d %10.1f %8.3f" % (ln, n, tot, tot / n))
    gaps.sort(reverse=True)
    print("idle gaps: %d, total %.1f ms; the 10 longest (ms, at ms):" % (len(gaps), sum(g for g, _ in gaps)), [(round(g, 2), round(t - t0, 1)) for g, t in gaps[:10]])
    hist = collections.Counter()
    for g, _ in gaps:
        hist["<0.05" if g < 0.05 else "<0.2" if g < 0.2 else "<1" if g < 1 else "<5" if g < 5 else ">=5"] += g
    print("idle time by gap length (ms):", {k: round(v, 1) for k, v in hist.items()})


if __name__ == "__main__":
    main()
