"""The attack-success table of the reference's experiment grid at C1, and what producing it costs.

The grid is tools/sweep_throughput.py's: MnistNet, N = 10 users, D = 79,510 fp32 at pitch --ld, z in {0.25, 0.5, 1.0,
1.5, 2.0, 3.0} x f in {1, 2} (Bulyan: f in {0, 1}) x S seeds, B = 12 S problems ordered cell by cell.  One round is
batched.alie_rows(G, f[], z[]), the rule on the whole batch, and then the success figures (SURVEY 8d): did Krum pick a
malicious user, which share of Bulyan's selection is malicious, and ||agg - honest_mean|| / ||honest_mean|| with the
honest mean over rows f_b..N-1 of each problem.  Three arms:
  rule     the attack and the rule only;
  device   the same, then one batched.attack_metrics call (no host synchronisation, Krum's rows read in place);
  looped   the same, then the per-problem loop over metrics.py: indices and selections copied to the host, one
           slice-mean and one relative_deviation (a host synchronisation) per problem.
Each arm is timed with CUDA events over --steps rounds after --warmup rounds, the arms alternate, --reps times, and the
median is reported in ms per round and aggregations/s (B problems per round).  In the same run, on a fresh copy of the
inputs, the device and looped figures must agree: flags and fractions equal, deviations within 1e-5 relative.  The
table has one row per (rule, z, f) cell, averaged over the seeds.  Prints one JSON object with the card's name and
power limit; fails without a GPU.

    python tools/sweep_report.py [--seeds 2,21] [--steps 10] [--warmup 2] [--reps 3] [--ld 79520] [--out FILE]
"""
import argparse
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import numpy as np  # noqa: E402
import torch  # noqa: E402

from host_outofcore import gpu_info  # noqa: E402
from sweep_throughput import D, N, RULES, ZS, fresh, grid, time_ms  # noqa: E402


def arms(bt, metrics, rule, G, S):
    _, f, z = grid(rule, S)
    B = G.shape[0]

    def attack_and_rule():
        """(aggregate [B, D] or None, Krum indices or None, Bulyan selections or None)"""
        bt.alie_rows(G, f, z)
        if rule == "Krum":
            return None, bt.krum(G, N, f, return_index=True), None
        if rule == "Bulyan":
            agg, sel = bt.bulyan(G, N, f, return_selection=True)
            return agg, None, sel
        return bt.defend[rule](G, N, f), None, None

    def device():
        agg, idx, sel = attack_and_rule()
        return bt.attack_metrics(G, f, aggregated=agg, krum_index=idx, selection=sel)

    def looped():
        agg, idx, sel = attack_and_rule()
        idx_h = None if idx is None else idx.cpu().tolist()
        sel_h = None if sel is None else sel.cpu().tolist()
        out = {"rel_deviation": [], "krum_success": [], "bulyan_malicious_fraction": []}
        for b in range(B):
            fb = int(f[b])
            honest = G[b, fb:].mean(0)
            a = G[b, idx_h[b]] if agg is None else agg[b]
            out["rel_deviation"].append(metrics.relative_deviation(a, honest))
            if idx_h is not None:
                out["krum_success"].append(metrics.krum_attack_success(idx_h[b], fb))
            if sel_h is not None:
                out["bulyan_malicious_fraction"].append(metrics.bulyan_attack_success(sel_h[b][:N - 2 * fb], fb))
        return out
    return {"rule": attack_and_rule, "device": device, "looped": looped}


def agree(dev, loop):
    """The device figures against the looped ones: flags and fractions equal, deviations within 1e-5 relative."""
    rel = np.asarray(dev["rel_deviation"].cpu().tolist())
    want = np.asarray(loop["rel_deviation"])
    ok = bool(np.all(np.abs(rel - want) <= 1e-5 * np.abs(want)))
    if loop["krum_success"]:
        ok = ok and dev["krum_success"].cpu().tolist() == loop["krum_success"]
    if loop["bulyan_malicious_fraction"]:
        got = dev["bulyan_malicious_fraction"].cpu().numpy()
        ok = ok and bool(np.array_equal(got, np.asarray(loop["bulyan_malicious_fraction"], np.float32)))
    return ok


def table(rule, S, dev):
    """One row per (z, f) cell: the seeds' mean of every figure attack_metrics returned."""
    cells, _, _ = grid(rule, S)
    rows = []
    for c, (z, f) in enumerate(cells):
        row = {"rule": rule, "z": z, "f": f}
        for key in ("rel_deviation", "krum_success", "bulyan_malicious_fraction"):
            if key in dev:
                row[key] = round(float(dev[key][c * S:(c + 1) * S].double().mean()), 6)
        rows.append(row)
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--seeds", default="2,21")
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--ld", type=int, default=79_520)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("sweep_report.py measures on a GPU; none is visible")
    from attacking_federate_learning_b200 import batched as bt, metrics
    info = {"gpu": gpu_info(), "device": torch.cuda.get_device_name(), "n": N, "d": D, "ld": a.ld, "z": ZS,
            "steps": a.steps, "warmup": a.warmup, "reps": a.reps, "timing": [], "success": []}
    for S in [int(x) for x in a.seeds.split(",")]:
        B = 12 * S
        gen = torch.Generator(device="cuda").manual_seed(1000 + S)
        buf = torch.empty((B, N, a.ld), dtype=torch.float32, device="cuda")
        buf.normal_(generator=gen)
        buf.mul_(torch.exp(0.25 * torch.randn((B, N, 1), device="cuda", generator=gen)))
        buf.add_(0.1 * torch.randn((B, 1, a.ld), device="cuda", generator=gen))    # the clients' common component
        G0 = buf[:, :, :D]
        for rule in RULES:
            dev = arms(bt, metrics, rule, fresh(G0), S)["device"]()
            ok = agree(dev, arms(bt, metrics, rule, fresh(G0), S)["looped"]())
            info["success"].append({"S": S, "rule": rule, "cells": table(rule, S, dev)})
            fns = arms(bt, metrics, rule, fresh(G0), S)
            for fn in fns.values():
                time_ms(fn, a.warmup)
            t = {k: [] for k in fns}
            for _ in range(a.reps):                                  # alternate the arms
                for k, fn in fns.items():
                    t[k].append(time_ms(fn, a.steps))
            med = {k: statistics.median(v) for k, v in t.items()}
            row = {"rule": rule, "S": S, "B": B, "device_agrees_with_looped": ok}
            for k in fns:
                row[f"{k}_ms"] = round(med[k], 4)
                row[f"{k}_aggs_per_s"] = round(B / med[k] * 1e3, 1)
                row[f"{k}_ms_all_reps"] = [round(x, 4) for x in t[k]]
            row["metrics_ms_device"] = round(med["device"] - med["rule"], 4)
            row["metrics_ms_looped"] = round(med["looped"] - med["rule"], 4)
            info["timing"].append(row)
            print(json.dumps(row), file=sys.stderr, flush=True)
        del buf, G0
        torch.cuda.empty_cache()
    info["agree_all"] = all(r["device_agrees_with_looped"] for r in info["timing"])
    text = json.dumps(info)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as fh:
            fh.write(text + "\n")
    print(text)
    if not info["agree_all"]:
        sys.exit("sweep_report.py: the device metrics disagree with the per-problem loop")


if __name__ == "__main__":
    main()
