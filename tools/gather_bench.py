"""Layer-0 fused gather + mean at the bench shape (5,632 output rows = 133,632 gathered rows): fp32 table vs bf16 table vs
int8 rows with a per-row scale (Int8Features: whole 608-byte rows at F = 602, scale included)."""
import os, sys
import numpy as np, torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import graphsage_b200 as gs
from graphsage_b200 import ops
dev = torch.device("cuda")
N, F, B = 232965, 602, 512
rs = np.random.RandomState(0)
tf = torch.zeros((N + 1, ops.pad_cols(F)), device=dev)
tf[:N, :F] = torch.randn((N, F), device=dev)
tb = tf.to(torch.bfloat16)
ti = gs.Int8Features(tf[:, :F])
import subprocess
print(subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                     text=True).stdout.strip())
sets = []
for i in range(6):
    s0 = torch.from_numpy(rs.randint(0, N, size=B).astype(np.int32)).to(dev)
    s1 = torch.from_numpy(rs.randint(0, N, size=B * 10).astype(np.int32)).to(dev)
    s2 = torch.from_numpy(rs.randint(0, N, size=B * 250).astype(np.int32)).to(dev)
    sets.append([ops.Seg(B, 10, self_ids=s0, neigh_ids=s1, out_row0=0), ops.Seg(B * 10, 25, self_ids=s1, neigh_ids=s2, out_row0=B)])
peak = 6572.5
for name, table, row_b in (("fp32 table", tf[:, :F], F * 4), ("bf16 table", tb[:, :F], F * 2), ("int8 rows", ti, ti.pitch)):
    for i in range(3):
        ops.gather_mean(table, sets[i])
    evs = []
    for i in range(24):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(); ops.gather_mean(table, sets[i % 6]); b.record()
        evs.append((a, b))
    torch.cuda.synchronize()
    t = float(np.median([a.elapsed_time(b) for a, b in evs])) * 1e3
    gb = B * 261 * row_b
    print("%s: %.1f us  algorithmic %.1f MB  %.0f GB/s = %.2f of the measured HBM peak (uniform random ids)" % (name, t, gb / 1e6, gb / t / 1e3, gb / t / 1e3 / peak))
