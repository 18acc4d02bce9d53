"""Per-kernel warp-stall summary from `ncu -i x.ncu-rep --page source --csv` (run the export ON the GPU box: the
reports themselves exceed gpurun's return limit).

    ncu -i conv.ncu-rep --page source --csv > gpurun_out/conv_source.csv          # on the box
    python tools/ncu_stalls.py gpurun_out/conv_source.csv r02a [top=12]            # here

writes profiles/<tag>_ncu_stalls.txt: for every captured launch the share of each stall reason over all sampled
instructions, and the `top` hottest SASS instructions with their own dominant reason -- the two things one reads
off the source page to decide what a wgmma / TMA kernel is waiting for (stall_long_sb = global loads in
flight, stall_barrier / stall_membar = mbarrier and fence waits, stall_no_inst = instruction fetch, ...).
"""
import csv
import io
import os
import re
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OUT_DIR = os.environ.get("NCU_SUMMARY_OUT", os.path.join(ROOT, "profiles"))


def sections(text):
    """[(kernel name, header, rows)] -- one per captured launch"""
    rows = list(csv.reader(io.StringIO(text)))
    out, i = [], 0
    while i < len(rows):
        r = rows[i]
        if len(r) >= 2 and r[0] == "Kernel Name":
            name = r[1]
            hdr = rows[i + 1] if i + 1 < len(rows) else []
            j = i + 2
            body = []
            while j < len(rows) and not (len(rows[j]) >= 2 and rows[j][0] == "Kernel Name"):
                if rows[j]:
                    body.append(rows[j])
                j += 1
            out.append((name, hdr, body))
            i = j
        else:
            i += 1
    return out


def num(x):
    try:
        return float(x.replace(",", ""))
    except ValueError:
        return 0.0


def summarise(name, hdr, body, top):
    col = {h: k for k, h in enumerate(hdr)}
    stall_cols = [h for h in hdr if h.startswith("stall_") and "(Not Issued)" not in h]
    samp = col.get("# Samples", col.get("Warp Stall Sampling (All Samples)"))
    src = col.get("Source")
    tot = {h: 0.0 for h in stall_cols}
    lines = []
    for r in body:
        if len(r) < len(hdr):
            continue
        for h in stall_cols:
            tot[h] += num(r[col[h]])
        n = num(r[samp]) if samp is not None else 0.0
        if n > 0:
            dom = max(stall_cols, key=lambda h: num(r[col[h]])) if stall_cols else "-"
            lines.append((n, r[src].strip() if src is not None else "?", dom, num(r[col[dom]]) if stall_cols else 0.0))
    all_s = sum(tot.values()) or 1.0
    short = re.sub(r"^(void )?mapnet::", "", name)
    short = re.sub(r"\(.*$", "", short)
    out = ["## %s   (%d SASS instructions, %d stall samples)" % (short, len(body), int(all_s))]
    out.append("   " + "  ".join("%s %.1f%%" % (h.replace("stall_", ""), 100.0 * v / all_s)
                                 for h, v in sorted(tot.items(), key=lambda kv: -kv[1])[:8] if v > 0))
    lines.sort(key=lambda t: -t[0])
    nsum = sum(t[0] for t in lines) or 1.0
    for n, s, dom, dn in lines[:top]:
        out.append("   %5.1f%%  %-60s %s %.0f%%" % (100.0 * n / nsum, s[:60], dom.replace("stall_", ""), 100.0 * dn / max(n, 1.0)))
    return "\n".join(out)


def main():
    path, tag = sys.argv[1], sys.argv[2]
    top = 12
    for a in sys.argv[3:]:
        if a.startswith("top="):
            top = int(a[4:])
    secs = sections(open(path).read())
    text = ["# warp-stall summary of %d captured launches (ncu --page source --csv; tools/ncu_stalls.py)" % len(secs)]
    for name, hdr, body in secs:
        text.append(summarise(name, hdr, body, top))
    out = os.path.join(OUT_DIR, "%s_ncu_stalls.txt" % tag)
    with open(out, "w") as f:
        f.write("\n\n".join(text) + "\n")
    print("wrote", out, len(secs), "launches")


if __name__ == "__main__":
    main()
