"""Pipeline timeline of CTA 0 (tiles 6..8) of the fused kernel from the test-only event trace.

usage: python scripts/trace_timeline.py [posterior|score]
Prints one line per event (SM clocks since the first one), then per warpgroup the clocks per tile, the share of the
tile spent in the chunk loop, the length of its MMA turns, and how many of one warpgroup's gaps between MMA turns (kernel values and epilogue on the
CUDA cores) see the other warpgroup issue its MMAs."""
import ctypes as C, sys
from pathlib import Path
sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
import torch
from baybe_b200 import AcqConfig, DeviceGP, sobol_normal_samples, _lib
from baybe_b200.synthetic import numeric_grid_workload

mode = sys.argv[1] if len(sys.argv) > 1 else "posterior"
dev = torch.device("cuda", 0)
w = numeric_grid_workload(N=1_000_000, d=20, n=256)
gp = DeviceGP(device=dev, **w.gp_kwargs())
x = torch.from_numpy(w.candidates).to(dev, torch.float32)
z = sobol_normal_samples(512, 1, 1234)[:, 0]
acq = AcqConfig(kind="qLogEI", best_f=gp.best_f(AcqConfig(kind="qLogEI")))
run = (lambda: gp.posterior(x)) if mode == "posterior" else (lambda: gp.score(acq, x, z, want_scores=False))
for _ in range(2): run()
torch.cuda.synchronize()
cap = 4000
buf = torch.zeros(1 + 2 * cap, dtype=torch.int64, device=dev)
lib = _lib.load()
lib.bb_debug_set_trace(C.c_void_p(buf.data_ptr()), cap)
run(); torch.cuda.synchronize()
lib.bb_debug_set_trace(None, 0)
h = buf.cpu()
n = min(int(h[0]), cap)
ev = sorted((int(h[2 + 2 * i]), int(h[1 + 2 * i])) for i in range(n))
if not ev:
    sys.exit("no trace events recorded")
t0 = ev[0][0]
# event ids of k_fused (fused_common.cuh): tile * 1000 + 100 * warpgroup + id
names = {0: "tile start", 1: "chunk loop done", 2: "epilogue done", 10: "MMA turn begin", 11: "MMA turn end"}
per_wg = {}
for clk, code in ev:
    it, r = divmod(code, 1000)
    wg, e = divmod(r, 100)
    per_wg.setdefault(wg, []).append((clk, it, e))
    print(f"{clk - t0:8d}  tile {it}  wg {wg}  {names.get(e, str(e))}")


def turns(evs):
    out, start = [], None
    for clk, _, e in evs:
        if e == 10:
            start = clk
        elif e == 11 and start is not None:
            out.append((start, clk))
            start = None
    return out


def covered(gaps, other):
    return sum(1 for a, b in gaps if any(a <= o0 < b for o0, _ in other))


for wg, evs in sorted(per_wg.items()):
    starts = {it: clk for clk, it, e in evs if e == 0}
    loops = {it: clk for clk, it, e in evs if e == 1}
    ends = {it: clk for clk, it, e in evs if e == 2}
    its = sorted(i for i in starts if i in ends)
    tile = [ends[i] - starts[i] for i in its]
    loop = [loops[i] - starts[i] for i in its if i in loops]
    if tile:
        print(f"wg {wg}: clocks per tile {sum(tile) / len(tile):.0f}, chunk loop {sum(loop) / max(1, len(loop)):.0f}, "
              f"epilogue {sum(tile) / len(tile) - sum(loop) / max(1, len(loop)):.0f}")
if len(per_wg) == 2:
    t0s, t1s = turns(per_wg[0]), turns(per_wg[1])
    lo = max(min(c for c, _, _ in per_wg[0]), min(c for c, _, _ in per_wg[1]))
    hi = min(max(c for c, _, _ in per_wg[0]), max(c for c, _, _ in per_wg[1]))
    for wg, mine, other in ((0, t0s, t1s), (1, t1s, t0s)):
        # gaps between my turns = time on the CUDA cores (kernel values, epilogue) or waiting
        gaps = [(a1, b0) for (_, a1), (b0, _) in zip(mine, mine[1:]) if lo <= a1 and b0 <= hi]
        if mine:
            print(f"wg {wg}: {len(mine)} MMA turns (granted -> MMAs issued), mean {sum(b - a for a, b in mine) / len(mine):.0f} "
                  f"clocks, longest {max(b - a for a, b in mine)}")
        if gaps:
            print(f"wg {wg}: {len(gaps)} gaps between its MMA turns, mean {sum(b - a for a, b in gaps) / len(gaps):.0f} "
                  f"clocks; the other warpgroup issues MMAs inside {covered(gaps, other)} of them")
