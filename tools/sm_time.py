#!/usr/bin/env python
"""SM-time view of ONE training step from an `ncu --metrics gpu__time_duration.sum` launch list (csv or csv.gz):
per kernel family the summed durations and the same weighted by the share of the GPU the launch can hold
(grid / (132 x CTAs per SM of that kernel)). If the weighted sum is close to the measured step time the step is bound by
SM occupancy (every launch that takes the whole GPU excludes the other streams), not by launch rate or by any single
chain's latency. usage: python tools/sm_time.py launches.csv.gz"""
import collections
import csv
import gzip
import re
import sys

path = sys.argv[1]
op = gzip.open if path.endswith(".gz") else open
with op(path, "rt") as f:
    lines = [l for l in f if not l.startswith("==")]
r = csv.reader(lines)
hdr = next(r)
ix = {h: i for i, h in enumerate(hdr)}
data = list(r)
names = [d[ix["Kernel Name"]] for d in data]
start = max(i for i, nm in enumerate(names) if "pack_weights" in nm and i < len(names) - 100)
step = data[start:]


def prod(field, d):
    n = 1
    for x in re.findall(r"\d+", d[ix[field]]):
        n *= int(x)
    return n


def share(nm, grid, block):
    if "halo_kernel<2" in nm or "igemm_kernel<2" in nm:      # two co-resident CTAs fill an SM (registers, shared memory)
        return min(1.0, grid / 264.0)
    if "halo_kernel<1" in nm or "conv_igemm_kernel<1" in nm or "wgrad_igemm" in nm:   # one CTA owns its SM
        return min(1.0, grid / 132.0)
    return min(1.0, grid / (132.0 * max(1, 2048 // block)))  # thread-slot share of the CUDA-core kernels


agg = collections.defaultdict(lambda: [0, 0.0, 0.0])
for d in step:
    nm = re.sub(r"\(.*", "", d[ix["Kernel Name"]]).replace("b200seg::", "").replace("void ", "")[:44]
    us = float(d[ix["Metric Value"]].replace(",", "")) / 1e3
    a = agg[nm]
    a[0] += 1
    a[1] += us
    a[2] += us * share(nm, prod("Grid Size", d), prod("Block Size", d))
tot, wtot = sum(a[1] for a in agg.values()), sum(a[2] for a in agg.values())
print("one step: %d launches, %.1f ms of serialised kernel time, %.1f ms weighted by the share of the GPU each launch holds"
      % (len(step), tot / 1e3, wtot / 1e3))
print("%-46s %5s %9s %11s %8s %9s" % ("kernel", "n", "sum ms", "SM-time ms", "avg us", "avg share"))
for k, a in sorted(agg.items(), key=lambda kv: -kv[1][2])[:18]:
    print("%-46s %5d %9.2f %11.2f %8.1f %9.2f" % (k, a[0], a[1] / 1e3, a[2] / 1e3, a[1] / a[0], a[2] / a[1]))
