"""L2 -> shared-memory fill rate of the forward / data-gradient convolutions' weight loads, per SM and in aggregate, with
and without 2-CTA TMA multicast (tools/l2_fill_bench.cu: a TMA producer streams an L2-resident weight tensor through a
shared-memory ring in the kernels' box shapes, a consumer releases each slot as soon as it lands). The Cout tile (BN)
and CTAs per SM of each shape are the ones b200seg_conv2d_plan_info picks for it. Compiles the benchmark with nvcc into a
temporary directory; the card's name, power limit and maximum SM clock are read in the same run. Bytes per clock are
per SM at the maximum SM clock.

--planes compares the halo kernel's two weight sources instead: 16-byte-row TMA planes of the [O][9][I] operand against
one contiguous 1-D bulk copy per plane of the plane-ordered image, at each Cout tile of PLANE_BN and the ring depth the
halo kernel plans for it, alternating the two modes --repeats times.

    python tools/gpu_l2_fill_bench.py [--tiles 4000] [--planes [--repeats 3]] [--out l2_fill.json]"""
import argparse
import ctypes
import json
import os
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "semantic-segmentation_b200"))

# (h, w, cin, cout, k) forward convolutions of the W48 step with streamed weights (one crop of 1024x2048)
SHAPES = [(256, 512, 720, 512, 3), (256, 512, 512, 256, 3), (256, 512, 1024, 512, 1), (256, 512, 720, 720, 1),
          (32, 64, 384, 384, 3), (16, 32, 384, 384, 3), (64, 128, 192, 192, 3)]
# (cin, cout) of the weight-streaming 3x3 layers of the W48 step, and the Cout tiles the planes comparison runs at
PLANE_SHAPES = [(720, 512), (512, 256), (256, 256)]
PLANE_BN = [256, 240, 128]


def halo_ring_slots(cout, bn):
    """(CTAs per SM, weight ring slots) of a weight-streaming halo launch with Cout tile bn: conv3x3_halo.cu's
    halo_smem_layout without a shared-memory reserve."""
    cout_pad = (cout + 15) // 16 * 16
    b_tile = (bn * 128 + 1023) // 1024 * 1024
    fixed = 1024 + (2 * 4 + 2 * 8) * 8 + 16 + 8 * 2 * cout_pad * 4
    for occ in ((2, 1) if bn <= 128 else (1,)):
        budget = (115712 if occ == 2 else 227 * 1024) - fixed
        slots = min(8, (budget - 2 * 24576) // b_tile)
        if slots >= (4 if occ == 2 else 2):
            return occ, slots
    raise ValueError("no halo ring for BN %d" % bn)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    return [s.strip() for s in q.split(",")]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--tiles", type=int, default=4000, help="weight tiles each CTA streams per launch")
    ap.add_argument("--planes", action="store_true", help="TMA planes against the plane-ordered image (halo kernel)")
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    from b200seg import _lib
    L = _lib.lib()
    nvcc = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin", "nvcc")
    tmp = tempfile.mkdtemp(prefix="l2_fill_")
    exe = os.path.join(tmp, "l2_fill_bench")
    subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-o", exe,
                    os.path.join(ROOT, "tools", "l2_fill_bench.cu")], check=True)
    name, power, clock = card()
    print("%s, power limit %s, max SM clock %s" % (name, power, clock))
    rows = []

    def run(kind, cin, cout, bn, occ, mc, slots=None):
        cmd = [exe, kind, str(cin), str(cout), str(bn), str(occ), str(mc), str(args.tiles)]
        out = subprocess.run(cmd + ([str(slots)] if slots else []), capture_output=True, text=True, timeout=300)
        if out.returncode:
            sys.exit(out.stderr)
        return json.loads(out.stdout.strip().splitlines()[-1])

    if args.planes:
        for (cin, cout) in PLANE_SHAPES:
            for bn in PLANE_BN:
                occ, slots = halo_ring_slots(cout, bn)
                for rep in range(args.repeats):
                    for kind in ("halo", "planes"):
                        r = run(kind, cin, cout, bn, occ, 0, slots)
                        r["repeat"] = rep
                        rows.append(r)
                        print("c%-4d->%-4d BN %3d occ %d slots %d %-6s #%d: smem fill %5.2f TB/s (%5.1f B/clk/SM)" % (
                            cin, cout, bn, occ, slots, kind, rep, r["smem_fill_TBps"], r["smem_fill_B_per_clk_per_sm"]),
                            flush=True)
        for (cin, cout) in PLANE_SHAPES:
            for bn in PLANE_BN:
                rate = {k: [r["smem_fill_TBps"] for r in rows if r["cin"] == cin and r["cout"] == cout and
                            r["BN"] == bn and r["kind"] == k] for k in ("halo", "planes")}
                print("c%d->%d BN %d: TMA planes %.2f-%.2f TB/s, image %.2f-%.2f TB/s, ratio of medians %.2f" % (
                    cin, cout, bn, min(rate["halo"]), max(rate["halo"]), min(rate["planes"]), max(rate["planes"]),
                    sorted(rate["planes"])[len(rate["planes"]) // 2] / sorted(rate["halo"])[len(rate["halo"]) // 2]))
    for (h, w, cin, cout, k) in ([] if args.planes else SHAPES):
        d = _lib.ConvDesc()
        d.n, d.h, d.w, d.cin, d.cout, d.ksize, d.stride, d.pad = 1, h, w, cin, cout, k, 1, (k - 1) // 2
        d.x_ld, d.y_ld, d.emit_stats = cin, cout, 1
        plan = (ctypes.c_int32 * 12)()
        assert L.b200seg_conv2d_plan_info(ctypes.byref(d), 0, plan) == 0, (h, w, cin, cout, k)
        kind, bn, occ = ("halo" if plan[0] == 1 else "igemm"), plan[1], plan[6]
        for mc in (0, 1):
            r = run(kind, cin, cout, bn, occ, mc)
            r["shape"] = "%dx%d c%d->%d k%d" % (h, w, cin, cout, k)
            rows.append(r)
            print("%-26s %-5s BN %3d occ %d %-9s grid %3d: smem fill %5.2f TB/s (%5.1f B/clk/SM), L2 read %5.2f TB/s "
                  "(%5.1f B/clk/SM)" % (r["shape"], kind, bn, occ, "multicast" if mc else "plain", r["grid"],
                                        r["smem_fill_TBps"], r["smem_fill_B_per_clk_per_sm"], r["l2_read_TBps"],
                                        r["l2_read_B_per_clk_per_sm"]), flush=True)
    if args.out:
        with open(args.out, "w") as f:
            json.dump(dict(card=dict(name=name, power_limit=power, max_sm_clock=clock), rows=rows), f, indent=1)


if __name__ == "__main__":
    main()
