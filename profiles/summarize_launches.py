#!/usr/bin/env python
"""Per-kernel shares of ONE training step from an ncu launch list
(`ncu --metrics gpu__time_duration.sum --clock-control none --csv --log-file X.csv python bench.py --steps 2 --warmup 3 ...`).

    python profiles/summarize_launches.py profiles/r2_launches_c2.csv

Durations are cold-cache and serialised: compare SHARES, not absolutes."""
import collections
import csv
import sys


def main(path):
    rows = list(csv.reader(open(path)))
    hdr = [i for i, r in enumerate(rows) if "Kernel Name" in r][0]
    cols = rows[hdr]
    ki, vi = cols.index("Kernel Name"), cols.index("Metric Value")
    recs = []
    for r in rows[hdr + 2:]:
        if len(r) > vi:
            try:
                recs.append((r[ki], float(r[vi].replace(",", ""))))
            except ValueError:
                pass
    # a step starts with the embedding gather; take the last complete one
    starts = [i for i, (n, _) in enumerate(recs) if "gather_uniform_fwd" in n or "embed_gather_generic" in n]
    st = [starts[0]]
    for i in starts[1:]:
        if i - st[-1] > 15:
            st.append(i)
    a, b = (st[-2], st[-1]) if len(st) >= 2 else (st[-1], len(recs))
    agg, n = collections.OrderedDict(), collections.Counter()
    for name, v in recs[a:b]:
        k = name.split("(")[0]
        agg[k] = agg.get(k, 0.0) + v
        n[k] += 1
    tot = sum(agg.values())
    print("%s: one step = %d launches, %.1f us serialised" % (path, b - a, tot / 1e3))
    for k, v in sorted(agg.items(), key=lambda kv: -kv[1]):
        print("  %-82s n=%3d %9.1f us %5.1f%%" % (k[:82], n[k], v / 1e3, 100 * v / tot))


if __name__ == "__main__":
    main(sys.argv[1])
