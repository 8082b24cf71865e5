"""ALIE z sweep (SURVEY 8d, Dist C) as one per-problem batch: problem i is the same client matrix attacked with z_i,
so one batched.alie_rows call replaces rows 0..f-1 of every problem by mu - z_i*sigma, and one batched Krum and one
batched Bulyan call aggregate them all.  Two batched.attack_metrics calls give the attack success of every z on the
device (Krum's rows are read in place); the host loop that follows only checks every problem's indices against the
NumPy oracle on the same inputs (Bulyan's sequence is required to match up to the first round whose top-1/top-2 margin
is below 1e-5).  The batched calls hold n <= 128 clients.
usage: python tools/attack_sweep.py [n] [d] > attack_sweep.json"""
import json, os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np, torch
from attacking_federate_learning_b200 import batched as bt
from oracle import ref_numpy as orc
import time

n = int(sys.argv[1]) if len(sys.argv) > 1 else 100
d = int(sys.argv[2]) if len(sys.argv) > 2 else 65536
if n > 128:
    sys.exit("attack_sweep.py runs the z sweep as one batch: n <= 128 clients")
f = int(0.24 * n)
zs = [0.25, 0.5, 1.0, 1.5, 2.0, 3.0]
rng = np.random.default_rng(2026)
base = (0.1 * rng.standard_normal(d) + rng.standard_normal((n, d)) * np.exp(0.25 * rng.standard_normal((n, 1)))).astype(np.float32)
Gd = torch.from_numpy(base).cuda().expand(len(zs), n, d).contiguous()
bt.alie_rows(Gd, f, zs)
k_dev = bt.krum(Gd, n, f, return_index=True)
agg, sel = bt.bulyan(Gd, n, f, return_selection=True)
by_krum = {key: v.cpu().tolist() for key, v in bt.attack_metrics(Gd, f, krum_index=k_dev).items()}
by_bulyan = {key: v.cpu().tolist() for key, v in bt.attack_metrics(Gd, f, aggregated=agg, selection=sel).items()}
k = k_dev.cpu().tolist()
torch.cuda.synchronize(); t0 = time.perf_counter()
for _ in range(3):
    bt.krum(Gd, n, f, return_index=True)
torch.cuda.synchronize(); t_krum = (time.perf_counter() - t0) / 3
t0 = time.perf_counter()
for _ in range(3):
    bt.bulyan(Gd, n, f)
torch.cuda.synchronize(); t_bulyan = (time.perf_counter() - t0) / 3
rows = []
for i, z in enumerate(zs):
    G = Gd[i].cpu().numpy()
    t64 = orc.pairwise_distances_f64(G)
    k_ref, margin = orc.krum_select(t64, orc.visit_order(n), n, f, dtype=np.float64, with_margin=True)
    sel_ref, margins = orc.bulyan_select(t64, n, f, dtype=np.float64, with_margins=True)
    first_close = next((j for j, m in enumerate(margins) if 0.0 < m <= 1e-5), len(margins))
    sel_l = sel[i].cpu().tolist()
    rows.append({"z": z, "krum_index": k[i], "krum_matches_oracle": k[i] == int(k_ref), "krum_margin": float(margin),
                 "krum_success": by_krum["krum_success"][i],
                 "bulyan_matches_oracle": sel_l[:first_close] == list(sel_ref)[:first_close],
                 "bulyan_rounds_required_exact": first_close, "bulyan_rounds": len(sel_l),
                 "bulyan_malicious_fraction": by_bulyan["bulyan_malicious_fraction"][i],
                 "bulyan_rel_deviation": by_bulyan["rel_deviation"][i],
                 "krum_rel_deviation": by_krum["rel_deviation"][i]})
# one batched call aggregates every z: aggregations/s counts problems
print(json.dumps({"n": n, "d": d, "f": f, "krum_aggregations_per_s": len(zs) / t_krum,
                  "bulyan_aggregations_per_s": len(zs) / t_bulyan, "sweep": rows}, indent=1))
