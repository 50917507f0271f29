#!/usr/bin/env python
"""Capacity planning without a GPU: weight arena and activation workspace of restore() for a batch shape, and the
largest batch that fits a given HBM budget (H100: 80 GB).  Uses the planning-only engine (vfx_engine_create with
device -1), i.e. the same dry-run allocator pass that sizes the workspace on the device.

    python tools/plan_capacity.py --seconds 10 --batch 32 --precision bf16 [--hbm-gb 80]
"""
import argparse
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def plan(seconds, batch, precision, hbm_gb=80.0, reserve_gb=4.0):
    from voicefixer_b200 import synthetic
    from voicefixer_b200.engine import Planner
    from voicefixer_b200.weights import pack_analysis, pack_vocoder
    packed = dict(pack_analysis(synthetic.make_analysis_state(0), precision), **pack_vocoder(synthetic.make_vocoder_state(1), precision))
    pl = Planner(packed, precision)
    L = int(round(seconds * 44100))
    io = lambda b: 2 * b * L * 4                                        # input + output waveforms on the device
    budget = (hbm_gb - reserve_gb) * 1e9 - pl.weight_bytes
    lo, hi = 1, 2
    while pl.workspace_bytes(hi, L) + io(hi) <= budget:
        lo, hi = hi, hi * 2
    while hi - lo > 1:
        mid = (lo + hi) // 2
        lo, hi = (mid, hi) if pl.workspace_bytes(mid, L) + io(mid) <= budget else (lo, mid)
    return {"precision": precision, "seconds": seconds, "batch": batch, "weights_gb": pl.weight_bytes / 1e9,
            "workspace_gb": pl.workspace_bytes(batch, L) / 1e9, "io_gb": io(batch) / 1e9,
            "per_item_gb": (pl.workspace_bytes(64, L) - pl.workspace_bytes(32, L)) / 32 / 1e9,
            "max_batch": lo, "hbm_gb": hbm_gb, "reserve_gb": reserve_gb}


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--seconds", type=float, default=10.0)
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--precision", default="bf16", choices=["bf16", "fp32"])
    ap.add_argument("--hbm-gb", type=float, default=80.0)
    a = ap.parse_args()
    for k, v in plan(a.seconds, a.batch, a.precision, a.hbm_gb).items():
        print(f"{k:14s} {v:.3f}" if isinstance(v, float) else f"{k:14s} {v}")
