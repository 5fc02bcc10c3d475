"""Per-phase cycle breakdown of the fused ct x ct kernel (DPFHE_KS_PROF build)."""
import os, sys, json
os.environ["DPFHE_KS_PROF"] = "1"
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch, time
import deeppowers_b200 as dp
log_n, L, B = 13, 4, 1184
c = dp.Context(log_n, L)
N = 1 << log_n
a = torch.empty((B, 2, L, N), dtype=torch.int64, device="cuda"); b = torch.empty_like(a); out = torch.empty_like(a)
evk = torch.empty((L, 2, L, N), dtype=torch.int64, device="cuda")
c.fill_uniform(1, a, 2 * B); c.fill_uniform(2, b, 2 * B); c.fill_uniform(3, evk, 2 * L)
c.ct_mul_relin(a, b, evk, out, B); c.phase_cycles()
c.ct_mul_relin(a, b, evk, out, B)
cyc = c.phase_cycles()
names = ["tensor+own key terms", "INTT register passes", "INTT outer stage + publish", "wait for sibling digit", "digit fetch + lift + outer fwd stage",
         "NTT register passes", "MAC with key column", "canon + store"]
items = B * L
tot = float(cyc[:8].sum())
print(json.dumps({"work_items": items, "cycles_per_item": tot / items,
                  "phases": {n: {"cycles_per_item": round(float(cyc[k]) / items), "share": round(float(cyc[k]) / tot, 3)} for k, n in enumerate(names)}}, indent=1))

# effective SM clock: cycles per round x rounds / wall time of the launch
import subprocess
e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
c.phase_cycles()
reps = 20
e0.record()
for _ in range(reps):
    c.ct_mul_relin(a, b, evk, out, B)
e1.record(); torch.cuda.synchronize()
ms = e0.elapsed_time(e1) / reps
cyc = c.phase_cycles()
grid = int(cyc[11])   # CTAs of the launched grid (the same in every launch of this shape)
smi = subprocess.run(["nvidia-smi", "--query-gpu=clocks.sm,power.draw,clocks_event_reasons.sw_power_cap", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
print(json.dumps({"grid_ctas": grid, "cta_ns_min_max": [float(cyc[12]) / reps, float(cyc[13]) / reps], "cta_ns_avg": float(cyc[14]) / reps / grid,
                  "cta_cycles_avg": float(cyc[15]) / reps / grid, "eff_mhz": float(cyc[15]) / float(cyc[14]) * 1e3, "ms_per_launch": ms,
                  "ct_per_s": B / ms * 1e3, "sum_cta_cycles_per_launch": float(cyc[:8].sum()) / reps, "smi_after": smi}))
