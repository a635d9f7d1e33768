#!/usr/bin/env python
"""GPU box: sampling-fraction learning (kl) of the CUDA path against the authors' logs and the oracle.
usage: learning_check.py [spaceship|kitchen] [repeats]"""
import json, os, sys, time
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "practical-path-guiding_b200")); sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np
import oracle_lib as O
from common import load_fixture_scene
from ppg_b200.integrator import GuidedPathTracer

what = sys.argv[1] if len(sys.argv) > 1 else "spaceship"
reps = int(sys.argv[2]) if len(sys.argv) > 2 else 2
with_oracle = (sys.argv[3] != "0") if len(sys.argv) > 3 else True
extra = dict(a.split("=") for a in sys.argv[1:] if "=" in a)
sys.argv = [a for a in sys.argv if "=" not in a]
if what == "cboxdef":
    sc = load_fixture_scene("cbox"); gold = []
elif what == "cbox":
    sc = load_fixture_scene("cbox-improved"); gold = json.load(open(os.path.join(ROOT, "tests", "golden", "cbox_log_stats.json")))["cbox-improved"]["iterations"]
elif what == "spaceship":
    sc = load_fixture_scene("spaceship-improved"); gold = json.load(open(os.path.join(ROOT, "tests", "golden", "spaceship_log_stats.json")))["spaceship-improved"]["iterations"]
else:
    sc = load_fixture_scene("kitchen-improved"); gold = json.load(open(os.path.join(ROOT, "tests", "golden", "kitchen_log_stats.json")))["kitchen-improved"]["iterations"]
budget = "63" if what == "spaceship" else "31"
if len(sys.argv) > 4: sc = sc.with_film(int(sys.argv[4]), int(sys.argv[4]))
props = dict(sc.integrator, budget=budget, **extra)
rows = []
for r in range(reps):
    g = GuidedPathTracer(dict(props, seed=str(1234 + r))); g.set_scene(sc)
    t = time.time(); img, st = g.render(); dt = time.time() - t
    rows.append(st["iterations"]); g.close()
    print("gpu run", r, "%.2fs" % dt, {k: round(v, 1) for k, v in st["kernel_ms"].items()}, "launches", st["kernel_launches"], "dropped", st["dropped_records"], "truncated", st["truncated_paths"], "sub-batches", st["sub_batches"], flush=True)
orow = None
if with_oracle:
    o = O.Oracle(O.params_from_xml(props), sc, kind="port"); t = time.time(); _, ost = o.render(); print("oracle %.1fs" % (time.time() - t)); orow = ost["iterations"]
print("iter | total weight (gpu runs.. | oracle | log) | leaves (gpu | oracle | log) | var (gpu | oracle | log)")
for k in range(len(rows[0])):
    gl = gold[k] if k < len(gold) else None
    tw = [it[k]["weight_avg"] * it[k]["s_tree_leaves"] for it in rows]
    lv = [it[k]["s_tree_leaves"] for it in rows]
    va = [it[k]["variance"] for it in rows]
    log_leaves = None
    print(k, "| W", ["%.0f" % x for x in tw], "| %s |" % ("%.0f" % (orow[k]["weight_avg"] * orow[k]["s_tree_leaves"]) if orow else "-"),
          "log avg %.1f" % gl["stat_weight"][1] if gl else "-", "| gpu avg", ["%.1f" % it[k]["weight_avg"] for it in rows], "oracle avg %.1f" % orow[k]["weight_avg"] if orow else "",
          "| L", lv, orow[k]["s_tree_leaves"] if orow else "-", "| V", ["%.4f" % x for x in va], "%.4f" % orow[k]["variance"] if orow else "-", gl["var"] if gl else "-", flush=True)
