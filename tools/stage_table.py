"""Per-stage view of the conv launches of ONE training step, from a committed launch list.

    python tools/stage_table.py profiles/h100_launches_raw.csv [peak_tflops] > profiles/h100_conv_by_stage.txt

The launch list (tools/profile_launches.py, torch.profiler's CUDA trace of one eager step of posenet_bs64; or
tools/launch_shares.py from an ncu capture) is in launch order, which is the trunk's schedule (geomapnet_b200/csrc/net.cu): forward = stem, then per
BasicBlock conv1, conv2[, downsample]; backward = blocks in reverse, per block dgrad(conv2) then dgrad(conv1) (a
downsampling block's conv1 dgrad carries the 1x1 shortcut dgrad in the same launch), wgrad(conv2), wgrad(conv1)
[, wgrad(downsample)], the stem's wgrad last.  Every conv launch is matched to its layer by position and its ALGORITHMIC
FLOPs (B = 64, 256x256) are divided by its duration.  Durations of an eager, traced step: compare stages with each other
and against bench.py's event-bracketed per-class numbers, not as absolute step time.  Default peaks: the H100 SXM data
sheet (989 dense bf16 TFLOP/s, 3350 GB/s HBM3), bounds that are not reached."""
import csv
import sys

B, HW = 64, 64          # frames, feature-map side after the stem pool (256x256 input)
STAGES = [(64, 3, 1), (128, 4, 2), (256, 6, 2), (512, 3, 2)]


def layers():
    stem = 2 * B * 128 * 128 * 64 * 147
    blocks, inpl, h = [], 64, HW
    for li, (pl, nb, st) in enumerate(STAGES):
        for b in range(nb):
            s = st if b == 0 else 1
            ho = h // s
            f1 = 2 * B * ho * ho * pl * 9 * inpl
            f2 = 2 * B * ho * ho * pl * 9 * pl
            fd = 2 * B * ho * ho * pl * inpl if (s != 1 or inpl != pl) else 0
            blocks.append(("layer%d" % (li + 1), f1, f2, fd))
            inpl, h = pl, ho
    return stem, blocks


def main():
    path = sys.argv[1]
    peak = float(sys.argv[2]) if len(sys.argv) > 2 else 989.0       # H100 SXM data sheet, dense bf16 TFLOP/s
    rows = list(csv.reader(open(path)))[1:]
    L = [(r[1], float(r[2]) / 1e3) for r in rows]                   # (kernel, us)
    stem, blocks = layers()
    split = next(i for i, (k, _) in enumerate(L) if k.startswith("k_gap_bwd"))
    fw = [x for x in L[:split] if x[0].startswith("k_tc_conv")]
    dg = [x for x in L[split:] if x[0].startswith("k_tc_conv")]
    wg = [x for x in L[split:] if x[0].startswith("k_tc_wgrad")]
    f_order = [("stem", stem)]
    for st, f1, f2, fd in blocks:
        f_order += [(st, f1), (st, f2)] + ([(st, fd)] if fd else [])
    d_order, w_order = [], []
    for st, f1, f2, fd in reversed(blocks):
        d_order += [(st, f2), (st, f1 + fd)]
        w_order += [(st, f2), (st, f1)] + ([(st, fd)] if fd else [])
    w_order.append(("stem", stem))
    assert len(fw) == len(f_order) == 36 and len(dg) == len(d_order) == 32 and len(wg) == len(w_order) == 36, \
        (len(fw), len(dg), len(wg))
    print("# %s: conv launches of one eager posenet_bs64 step by ResNet stage; peak = %.1f TFLOP/s" % (path, peak))
    grand_us = grand_fl = 0.0
    for name, lst, order in (("fprop", fw, f_order), ("dgrad", dg, d_order), ("wgrad", wg, w_order)):
        agg = {}
        for (k, us), (st, fl) in zip(lst, order):
            a = agg.setdefault(st, [0.0, 0.0, 0, set()])
            a[0] += us; a[1] += fl; a[2] += 1; a[3].add(k.split("(")[0])
        tu = sum(a[0] for a in agg.values()); tf = sum(a[1] for a in agg.values())
        grand_us += tu; grand_fl += tf
        print("\n%s | launches | us | GFLOP | TFLOP/s | of peak | share of %s time | share of FLOPs | kernels" % (name, name))
        for st in ("stem", "layer1", "layer2", "layer3", "layer4"):
            if st not in agg:
                continue
            us, fl, n, ks = agg[st]
            print("%-6s | %2d | %6.1f | %6.1f | %4.0f | %.2f | %4.1f %% | %4.1f %% | %s"
                  % (st, n, us, fl / 1e9, fl / us / 1e6, fl / us / 1e6 / peak, 100 * us / tu, 100 * fl / tf, ", ".join(sorted(ks))))
        print("%-6s | %2d | %6.1f | %6.1f | %4.0f | %.2f" % ("all", sum(a[2] for a in agg.values()), tu, tf / 1e9,
                                                          tf / tu / 1e6, tf / tu / 1e6 / peak))
    print("\nall conv launches: %.1f us, %.1f GFLOP, %.0f TFLOP/s = %.2f of peak"
          % (grand_us, grand_fl / 1e9, grand_fl / grand_us / 1e6, grand_fl / grand_us / 1e6 / peak))
    elementwise(L, split)


def elementwise(L, split, hbm=3350.0):
    """BatchNorm apply kernels by stage, against the HBM roofline in ALGORITHMIC bytes (bf16 tensors): forward
    k_bn_apply_lazy<.., RES> reads y [+ the residual or the downsample conv's output] and writes z: 4 / 6 / 6 bytes per
    element for RES = 0 / 1 / 2; backward k_bn_bwd_apply*<.., DS, ..> reads the (already ReLU-gated) gradient and y and
    writes dy: 6 bytes per element, 10 with the downsample BN's second input / output (DS = 1), +2 with a second gradient output (GO = 1).  Two launches per
    BasicBlock in each direction (+ the head-side one and the stem's in the backward)."""
    per_stage = [("layer1", 3, B * 64 * 64 * 64), ("layer2", 4, B * 32 * 32 * 128), ("layer3", 6, B * 16 * 16 * 256),
                 ("layer4", 3, B * 8 * 8 * 512)]
    fw = [x for x in L[:split] if x[0].startswith("k_bn_apply_lazy")]
    bw = [x for x in L[split:] if x[0].startswith("k_bn_bwd_apply")]
    f_order = [(st, el) for st, nb, el in per_stage for _ in range(2 * nb)]
    b_order = [(st, el) for st, nb, el in reversed(per_stage) for _ in range(2 * nb)] + [("stem", B * 128 * 128 * 64)]
    assert len(fw) == len(f_order) == 32 and len(bw) == len(b_order) == 33, (len(fw), len(bw))

    def bytes_per_elt(kernel, fwd):
        args = kernel[kernel.index("<") + 1:kernel.rindex(">")].split(",")
        if fwd:
            return 4 if int(args[2]) == 0 else 6
        return (10 if int(args[3]) == 1 else 6) + (2 if int(args[4]) == 1 else 0)      # GO = 1: a second gradient output

    for name, lst, order, fwd in (("BatchNorm apply, forward", fw, f_order, True), ("BatchNorm apply, backward", bw, b_order, False)):
        agg = {}
        for (k, us), (st, el) in zip(lst, order):
            a = agg.setdefault(st, [0.0, 0.0, 0])
            a[0] += us; a[1] += el * bytes_per_elt(k, fwd); a[2] += 1
        print("\n%s | launches | us | algorithmic MB | GB/s | of %.0f GB/s" % (name, hbm))
        tu = tb = 0.0
        for st in ("stem", "layer1", "layer2", "layer3", "layer4"):
            if st in agg:
                us, by, n = agg[st]
                tu += us; tb += by
                print("%-6s | %2d | %6.1f | %7.1f | %5.0f | %.2f" % (st, n, us, by / 1e6, by / us / 1e3, by / us / 1e3 / hbm))
        print("%-6s | %2d | %6.1f | %7.1f | %5.0f | %.2f" % ("all", sum(a[2] for a in agg.values()), tu, tb / 1e6, tb / tu / 1e3,
                                                            tb / tu / 1e3 / hbm))


if __name__ == "__main__":
    main()
