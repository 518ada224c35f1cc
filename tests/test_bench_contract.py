"""bench.py on the CPU: the workloads follow BASELINE.json's configs, the pair sharding is a partition, and the reference arm
(`--impl reference`, the CPU restatement on the host cores) prints a line with every key of the measurement contract."""
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def test_workloads_follow_baseline_configs():
    import bench
    base = json.load(open(os.path.join(ROOT, "BASELINE.json")))
    assert bench.METRIC.startswith("flow_residual_constraints_per_sec") and "constraints/sec" in base["metric"]
    wl = bench.WORKLOADS
    spec2 = wl["config2_300f_384x224_grid16x12_sep10"]
    assert (spec2["frames"], spec2["w"], spec2["h"], spec2["gx"], spec2["gy"], spec2["sep"]) == (300, 384, 224, 16, 12, 10)      # configs[1]
    assert wl["config3_300f_384x224_grid16x12_sep10_maskratio0.20"]["mask_ratio"] == 0.20                                       # configs[2]
    s4 = wl["config4_600f_640x384_grid32x24_sep10_huber"]
    assert (s4["frames"], s4["w"], s4["h"], s4["gx"], s4["gy"]) == (600, 640, 384, 32, 24) and s4["cfg"]["robust_type"] == bench.abi.ROBUST_HUBER   # configs[3]
    assert wl["config5_300f_384x224_grid16x12_sep10_holes50_dolly"]["scene"]["hole_fraction"] > 0                                # configs[4]
    # config 1 builds in a blink: records, pair list and medians have consistent shapes; the overlap filter and the holes act
    spec, sc, cfg, pairs, offs, rec, med = bench.build_case("config1_8f_128x96_grid4x4_sep10")
    assert rec.shape[1] == 6 and offs[-1] == rec.shape[0] and len(pairs) == len(offs) - 1 == 30 and med.shape == (8,)
    from robust_cvd_b200 import synthetic
    fast = synthetic.Scene(40, 128, 96, seed=2, rot_deg=6.0, motion=0.15)
    kept = fast.filtered_pairs(0.2)
    assert 0 < len(kept) < len(synthetic.hierarchical2_pairs(40)) and all(fast.mask_ratio(a, b) > 0.2 for a, b in kept[:5])
    holes = synthetic.Scene(6, 128, 96, seed=2, hole_fraction=0.29, dolly=0.008)
    py, px = np.mgrid[0:96, 0:128]
    assert 0.55 < holes.visible(3, px.ravel(), py.ravel()).mean() < 0.85
    assert holes.constraints(sep=10)[2].shape[0] < 0.8 * synthetic.Scene(6, 128, 96, seed=2, dolly=0.008).constraints(sep=10)[2].shape[0]


def test_pair_sharding_is_a_balanced_partition():
    import bench
    spec, sc, cfg, pairs, offs, rec, med = bench.build_case("config1_8f_128x96_grid4x4_sep10")
    seen = []
    counts = []
    for r in range(3):
        lp, lo, lr = bench.shard_pairs(pairs, offs, rec, r, 3)
        seen += [tuple(p) for p in lp]; counts.append(lr.shape[0])
        assert lo[-1] == lr.shape[0]
    assert sorted(seen) == sorted(tuple(p) for p in pairs) and sum(counts) == rec.shape[0]
    assert max(counts) - min(counts) <= np.diff(offs).max()


def test_reference_arm_prints_the_contract_line():
    """`bench.py --impl reference` needs no GPU: smallest workload, one step."""
    out = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--impl", "reference", "--workload", "config1_8f_128x96_grid4x4_sep10", "--steps", "1", "--warmup", "1"],
                         capture_output=True, text=True, timeout=600, cwd=ROOT)
    assert out.returncode == 0, out.stderr[-2000:]
    d = json.loads(out.stdout.strip().splitlines()[-1])
    for k in ("impl", "metric", "value", "unit", "n_gpus", "steps", "warmup", "ms_per_step", "higher_is_better", "scaling", "vs_baseline", "dtype", "data", "config", "cpu_baseline", "e2e"):
        assert k in d, k
    assert d["impl"] == "reference" and d["value"] > 0 and d["cpu_baseline"]["cores"] >= 1 and d["cpu_baseline"]["kind"] == "port" and d["config"]["workload"].startswith("config1")
    assert d["e2e"] == {"value": d["value"], "unit": d["unit"], "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0}
