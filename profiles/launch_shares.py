#!/usr/bin/env python
"""Per-kernel launch counts and device-time shares of one `ncu --metrics gpu__time_duration.sum --csv` launch
list (times under ncu are cold-cache and serialised: compare SHARES, not absolutes).
usage: python profiles/launch_shares.py x_launches.csv"""
import collections
import csv
import re
import sys

rows = [r for r in csv.reader(open(sys.argv[1], errors="replace")) if len(r) > 10 and r[0].isdigit()]
tot = collections.Counter()
cnt = collections.Counter()
for r in rows:
    name = re.sub(r"\(.*", "", r[4]).replace("void ", "").replace("dfgpu::", "")
    ns = float(r[-1].replace(",", ""))
    unit = r[-2]
    us = ns / 1e3 if unit in ("ns", "nsecond") else (ns if unit in ("us", "usecond") else ns * 1e3)
    tot[name] += us
    cnt[name] += 1
total = sum(tot.values())
print("%d launches, %.1f ms of device time" % (len(rows), total / 1e3))
print("%-60s %8s %12s %8s %10s" % ("kernel", "launches", "total us", "share", "avg us"))
for k, v in tot.most_common():
    print("%-60s %8d %12.1f %7.1f%% %10.1f" % (k[:60], cnt[k], v, 100 * v / total, v / cnt[k]))
