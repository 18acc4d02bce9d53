"""The numbers the documents quote are the numbers of the committed evidence (CPU only, no compute).

README.md, DESIGN.md and profiles/README.md quote bench lines; every quoted figure must be readable from a file under
profiles/, which also records the GPU the line was measured on."""
import json
import os
import re

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PROF = os.path.join(ROOT, "profiles")


def _line(name):
    with open(os.path.join(PROF, name)) as f:
        return json.loads([l for l in f.read().splitlines() if l.startswith("{")][0])


def _fmt(v):
    """17107.26 -> '17 107' (the thin-space thousands style the documents use)."""
    s = "%d" % round(v)
    return s if len(s) <= 3 else s[:-3] + " " + s[-3:]


BENCH = {
    "posenet_bs64": "h100_bench_posenet_bs64.json",
    "mapnet_n32t3": "h100_bench_mapnet_n32t3.json",
    "mapnetpp_n16t10": "h100_bench_mapnetpp_n16t10.json",
}


def test_readme_and_design_quote_the_committed_bench_lines():
    readme = open(os.path.join(ROOT, "README.md")).read()
    design = open(os.path.join(ROOT, "DESIGN.md")).read()
    prof = open(os.path.join(PROF, "README.md")).read()
    for key, fn in BENCH.items():
        d = _line(fn)
        assert d["config"]["workload"] == key and d["n_gpus"] == 1
        assert "H100" in open(os.path.join(PROF, fn)).read().splitlines()[0]
        for doc_name, doc in (("README.md", readme), ("DESIGN.md", design), ("profiles/README.md", prof)):
            assert _fmt(d["value"]) in doc, (doc_name, key, _fmt(d["value"]))
            assert _fmt(d["e2e"]["value"]) in doc, (doc_name, key, "e2e", _fmt(d["e2e"]["value"]))
    d = _line(BENCH["posenet_bs64"])
    # a throttled measurement is only quoted together with the throttle and the power limit it ran at
    if d["clocks"]["reasons"] != []:
        head = open(os.path.join(PROF, BENCH["posenet_bs64"])).read().splitlines()[0]
        assert "sw_power_cap" in head and "power limit" in head and "power cap" in readme and "power limit" in design
    assert d["e2e"]["h2d_bytes_per_step"] == 64 * 3 * 256 * 256 * 4 + 64 * 6 * 4
    # the roofline fraction README states, against the data-sheet peak recorded in the line
    assert d["roofline"]["peak"] == 989.0 and ("%.3f" % d["roofline"]["frac"]) in readme and ("%.3f" % d["roofline"]["frac"]) in design
    # both tensor-core modes were measured in the same run
    pm = d["precision_modes"]
    assert pm["bf16"]["images_per_s"] == d["value"]
    assert ("%.2f k" % (pm["tc_split"]["images_per_s"] / 1000.0)) in readme and ("%.2f k" % (pm["tc_split"]["images_per_s"] / 1000.0)) in design
    assert ("%.1f" % d["cpu_baseline"]["value"]) in readme


def test_bench_note_cites_an_existing_file():
    src = open(os.path.join(ROOT, "bench.py")).read()
    for m in re.finditer(r"profiles/[A-Za-z0-9_]+\.json", src):
        assert os.path.exists(os.path.join(ROOT, m.group(0))), m.group(0)


def test_stage_table_accounts_for_every_conv_flop_of_the_step():
    """tools/stage_table.py matches the 104 conv launches of the committed launch list to their layers: the algorithmic
    FLOPs must add up to SURVEY.md 8d's per-step figure (B = 64: 1 817.6 GFLOP), and the committed table is its output."""
    import subprocess
    import sys
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "stage_table.py"),
                        os.path.join("profiles", "h100_launches_raw.csv")], capture_output=True, text=True, cwd=ROOT, timeout=120)
    assert r.returncode == 0, r.stderr
    assert "1817.6 GFLOP" in r.stdout and "all    | 36 |" in r.stdout and "all    | 32 |" in r.stdout
    assert r.stdout == open(os.path.join(PROF, "h100_conv_by_stage.txt")).read()
    from oracle import mapnet_oracle as O
    assert abs(64 * O.train_flops_per_image(256, 256) - 1817.6e9) < 0.1e9
