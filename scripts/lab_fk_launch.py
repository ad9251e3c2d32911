#!/usr/bin/env python
"""A/B lab for the FK+Jacobian launch at the contract batch (Kuka iiwa, 65 536 configurations per launch).

For every kernel variant (CTA-tile kernel vs per-warp pipeline kernel, warps per CTA, programmatic dependent launch
mode) it reports
  serial_us     per launch, CUDA graph of 64 kernel nodes on ONE stream (strictly stream-ordered launches)
  branch4_us    per launch, the same 64 nodes in 4 parallel graph branches (independent batches in flight)
  isolated_us   one launch between two events after an L2 flush (includes the event / launch gap; compare, don't quote)
  big_us        one launch of 2^22 configurations
and checks that every variant is BIT-identical to the first.  Prints one JSON object."""
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import differentiable_robot_model_b200 as drm  # noqa: E402
from differentiable_robot_model_b200 import engine  # noqa: E402

DEV = torch.device("cuda", 0)
BYTES = 224
OPTS = ("fk_kernel", "fk_tile", "fk_warps", "fk_pdl", "fk_grid_cap")


def set_opts(d):
    base = {"fk_kernel": 0, "fk_tile": 0, "fk_warps": 0, "fk_pdl": 0, "fk_grid_cap": 0}
    base.update(d)
    for k in OPTS:
        engine.set_option(k, base[k])


def main():
    m = drm.DifferentiableKUKAiiwa(device=DEV)
    table, topo, ee = m._link_table(), m._topology, m._name_to_idx_map["iiwa_link_ee"]
    small, big, R = 65536, 1 << 22, 16
    gen = torch.Generator(device="cpu").manual_seed(0)
    qs = [((torch.rand(small, 7, generator=gen) * 2 - 1) * 2.9).to(DEV) for _ in range(R)]
    outs = [(torch.empty(small, 3, device=DEV), torch.empty(small, 4, device=DEV), torch.empty(small, 3, 7, device=DEV),
             torch.empty(small, 3, 7, device=DEV)) for _ in range(R)]
    q_big = torch.cat(qs * (big // small // R))
    out_big = (torch.empty(big, 3, device=DEV), torch.empty(big, 4, device=DEV), torch.empty(big, 3, 7, device=DEV),
               torch.empty(big, 3, 7, device=DEV))
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=DEV)
    stream = torch.cuda.Stream(device=DEV)
    variants = [
        {"fk_kernel": 0, "fk_tile": 128, "fk_pdl": 0},
        {"fk_kernel": 0, "fk_tile": 64, "fk_pdl": 0},
        {"fk_kernel": 0, "fk_tile": 128, "fk_pdl": 2},
        {"fk_kernel": 0, "fk_tile": 64, "fk_pdl": 2},
        {"fk_kernel": 0, "fk_tile": 256, "fk_pdl": 2},
        {"fk_kernel": 0, "fk_tile": 128, "fk_pdl": 1},
        {"fk_kernel": 1, "fk_warps": 4, "fk_pdl": 0},
        {"fk_kernel": 1, "fk_warps": 4, "fk_pdl": 2},
        {"fk_kernel": 1, "fk_warps": 8, "fk_pdl": 2},
    ]
    only = os.environ.get("LAB_VARIANTS")
    if only:
        variants = [variants[int(i)] for i in only.split(",")]
    rows, ref = [], None
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for v in variants:
        set_opts(v)
        row = dict(v)
        with torch.cuda.stream(stream):
            got = engine.fk_jacobian_raw(topo, ee, table, qs[0])
            ragged = engine.fk_jacobian_raw(topo, ee, table, qs[1][:4099])
            stream.synchronize()
            got = [t.clone() for t in got] + [t.clone() for t in ragged]
            if ref is None:
                ref = got
                expected = [[t.clone() for t in engine.fk_jacobian_raw(topo, ee, table, qs[i])] for i in range(R)]
                stream.synchronize()
            row["bit_identical_to_first"] = all(torch.equal(a, b) for a, b in zip(ref, got))
            # large batch
            for _ in range(3):
                engine.fk_jacobian_raw(topo, ee, table, q_big, out=out_big)
            e0.record(stream)
            for _ in range(10):
                engine.fk_jacobian_raw(topo, ee, table, q_big, out=out_big)
            e1.record(stream)
            stream.synchronize()
            ms = e0.elapsed_time(e1) / 10
            row["big_us"] = ms * 1e3
            row["big_frac_of_3350"] = big * BYTES / ms / 1e6 / 3350.0     # H100 SXM data-sheet HBM3 GB/s
            # isolated launches after an L2 flush
            iso = []
            for i in range(12):
                flush.fill_(i)
                stream.synchronize()
                e0.record(stream)
                engine.fk_jacobian_raw(topo, ee, table, qs[i % R], out=outs[i % R])
                e1.record(stream)
                stream.synchronize()
                iso.append(e0.elapsed_time(e1) * 1e3)
            row["isolated_us_median"] = sorted(iso[2:])[len(iso[2:]) // 2]
            for inflight in (1, 2, 4):
                side = [torch.cuda.Stream(device=DEV) for _ in range(inflight - 1)]
                stream.synchronize()
                g = torch.cuda.CUDAGraph()
                nodes = 64
                with torch.cuda.graph(g, stream=stream):
                    fork = torch.cuda.Event()
                    fork.record(stream)
                    for s in side:
                        s.wait_event(fork)
                    for i in range(nodes):
                        lane = i % inflight
                        if lane == 0:
                            engine.fk_jacobian_raw(topo, ee, table, qs[i % R], out=outs[i % R])
                        else:
                            with torch.cuda.stream(side[lane - 1]):
                                engine.fk_jacobian_raw(topo, ee, table, qs[i % R], out=outs[i % R])
                    for s in side:
                        j = torch.cuda.Event()
                        j.record(s)
                        stream.wait_event(j)
                for _ in range(3):
                    g.replay()
                stream.synchronize()
                samples = []
                for _ in range(7):
                    e0.record(stream)
                    for _ in range(20):
                        g.replay()
                    e1.record(stream)
                    stream.synchronize()
                    samples.append(e0.elapsed_time(e1) * 1e3 / (20 * nodes))
                us = sorted(samples)[3]
                key = "serial" if inflight == 1 else f"branch{inflight}"
                row[f"{key}_us"] = us
                row[f"{key}_outputs_ok"] = all(torch.equal(a, b) for i in range(R) for a, b in zip(expected[i], outs[i]))
                for o in outs:
                    for t in o:
                        t.zero_()
                row[f"{key}_frac_of_3350"] = small * BYTES / us / 1e3 / 3350.0
                del g
        rows.append(row)
        print(json.dumps(row), file=sys.stderr, flush=True)
    set_opts({})
    print(json.dumps({"gpu": torch.cuda.get_device_name(0), "batch": small, "rows": rows}))


if __name__ == "__main__":
    main()
