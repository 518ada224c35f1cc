"""Memory-traffic model of the block-Cholesky Schur updates (k_update_tma, robust_cvd_b200/csrc/rcvd_update.cuh), from the plan alone:
no GPU.  python tools/update_traffic.py [--configs 2 4 5] [--order 0|1|both] [--launches]

An item streams, for each of its source pairs, an mrows-row strip of X_rk and an ncols-row strip of X_ck (the TMA fetches whole
16-column stages: ceil(neff / 16) * 16 doubles per row), then reads and writes its target tile.  The factor is far larger than the
H100's 50 MB L2, so a strip is an L2 hit only if an item running at about the same time read it: a wave is `ctas` consecutive items
(the persistent CTAs take items b, b + ctas, ...).  Per launch the model prints:
  items, waves (items / resident CTAs), streamed operand bytes, unique operand bytes (distinct (T block, strip) pairs), the largest
  per-wave unique operand bytes, the estimated operand bytes from HBM (a strip is a miss in a wave unless the same or the previous
  wave used it), and the target read-modify-write bytes.
All of these are counts from the plan; the HBM figure is an estimate of what the L2 has to fetch, not a measurement."""
import argparse
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np

from robust_cvd_b200 import abi, solver, synthetic

# the structure of bench.py's workloads: hierarchical2 pairs, a bilinear depth grid (gx x gy)
CONFIGS = {2: dict(frames=300, gx=16, gy=12), 4: dict(frames=600, gx=32, gy=24), 5: dict(frames=300, gx=16, gy=12)}
H100_SMS = 132


def plan_items(config, order, num_sms=H100_SMS):
    spec = CONFIGS[config]
    cfg = abi.default_config(spec["frames"], 384 / 224, depth_type=abi.DEPTH_GRID, depth_grid_x=spec["gx"], depth_grid_y=spec["gy"])
    return solver.update_items(cfg, synthetic.hierarchical2_pairs(spec["frames"]), num_sms=num_sms, order=order)


def launch_traffic(items, products, kbytes, ctas):
    """Model of one launch (items: [n, 8] in launch order)."""
    n = items.shape[0]
    dst, first, count, m0, n0, mrows, ncols, flags = items.T.astype(np.int64)
    rep = np.repeat(np.arange(n), count)
    pair = first[rep] + (np.arange(rep.size) - np.repeat(np.cumsum(count) - count, count))
    wave = rep // ctas
    # strips: (T block, first row); the A strip of an item is X_rk rows m0.., the B strip X_ck rows n0.. (one T buffer)
    key = np.concatenate([products[pair, 0] * 4096 + m0[rep], products[pair, 1] * 4096 + n0[rep]])
    rows = np.concatenate([mrows[rep], ncols[rep]])
    wv = np.concatenate([wave, wave])
    streamed = int(rows.sum()) * kbytes
    uk, ui = np.unique(key, return_index=True)
    unique = int(rows[ui].sum()) * kbytes
    big = np.int64(1) << 40
    wk, wi = np.unique(wv * big + key, return_index=True)
    wsize = rows[wi] * kbytes
    per_wave = np.bincount(wk // big, weights=wsize)
    hit_prev = np.isin(wk - big, wk)                      # the same strip in the previous wave
    hbm = int(wsize[~hit_prev].sum())
    hm = ((mrows // 8 + 1) // 2) * 8
    hn = ((ncols // 8 + 1) // 2) * 8
    area = mrows * ncols - np.where(flags & 1, hm * (ncols - hn), 0)
    rmw = int((area * 8 * np.where(flags & 2, 1, 2)).sum())
    return dict(items=n, ctas=ctas, waves=n / ctas, streamed=streamed, unique=unique, wave_unique_max=float(per_wave.max()),
                wave_unique_mean=float(per_wave.mean()), hbm=hbm, rmw=rmw)


def model(config, order, num_sms=H100_SMS):
    """Per launch (level, launch: 0 late, 1 / 2 deferred) the traffic of the plan's update items at `config` in `order`."""
    P = plan_items(config, order, num_sms)
    kbytes = (P["neff"] + 15) // 16 * 16 * 8
    out = []
    for lvl, ls in enumerate(P["launches"]):
        for s, (off, n) in enumerate(ls):
            if n == 0:
                continue
            ctas = n if n <= num_sms else min(n, 2 * num_sms)    # rcvd_update.cuh upd_ctas
            out.append(dict(level=lvl, launch=s, **launch_traffic(P["items"][off:off + n], P["products"], kbytes, ctas)))
    return out


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--configs", type=int, nargs="+", default=[2, 4, 5], choices=sorted(CONFIGS))
    ap.add_argument("--order", default="both", choices=["0", "1", "both"], help="0: cost-sorted, 1: locality order (the default)")
    ap.add_argument("--launches", action="store_true", help="print every launch, not only the totals")
    a = ap.parse_args()
    MB = 1e6
    for c in a.configs:
        for order in ([0, 1] if a.order == "both" else [int(a.order)]):
            rows = model(c, order)
            name = "locality" if order else "cost-sorted"
            if a.launches:
                print(f"config {c}, {name} order: level launch items ctas waves | streamed unique wave-unique(max, mean) HBM-est RMW [MB]")
                for r in rows:
                    print(f"  {r['level']:3d} {r['launch']} {r['items']:6d} {r['ctas']:4d} {r['waves']:6.1f} | {r['streamed'] / MB:9.1f} {r['unique'] / MB:8.1f} "
                          f"{r['wave_unique_max'] / MB:7.1f} {r['wave_unique_mean'] / MB:7.1f} {r['hbm'] / MB:9.1f} {r['rmw'] / MB:8.1f}")
            multi = [r for r in rows if r["waves"] > 1]
            tot = {k: sum(r[k] for r in rows) for k in ("items", "streamed", "unique", "hbm", "rmw")}
            wmax = max((r["wave_unique_max"] for r in multi), default=0.0)
            wmean = sum(r["wave_unique_mean"] * r["waves"] for r in multi) / max(sum(r["waves"] for r in multi), 1e-9)
            print(f"config {c}, {name} order: {len(rows)} launches ({len(multi)} of several waves), {tot['items']} items; operand bytes "
                  f"streamed {tot['streamed'] / MB:.0f} MB, unique {tot['unique'] / MB:.0f} MB, estimated from HBM {tot['hbm'] / MB:.0f} MB; "
                  f"per-wave unique operand bytes (multi-wave launches) mean {wmean / MB:.1f} MB, max {wmax / MB:.1f} MB; "
                  f"target read-modify-write {tot['rmw'] / MB:.0f} MB")


if __name__ == "__main__":
    main()
