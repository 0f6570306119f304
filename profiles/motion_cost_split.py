"""Learned edge cost of whole edges and paths (artp_motion_cost_split[_device]) against the head alone and the per-edge path.

For 100 k edges from synth.make_edges (0.5-2 m, 2-5 pieces each) on the 256 x 256 patch and on the 1000 x 1000 map:
  * split device call (rows + head + reduce) and artp_motion_cost_device over the same pieces, CUDA events, >= 20 calls;
  * the host entry point end to end (staging copies included);
  * per-edge baselines over 2 000 edges: motionCost (one host call per edge), and costQuery of the edge's own rows
    (one artp_motion_cost call per edge, what the C++ mirror's per-edge motionCost makes);
  * pathCost of a 300-state path as one batch against 299 per-edge calls.
Prints the GPU name, power limit and max SM clock first: the numbers mean nothing without them.

    python profiles/motion_cost_split.py [--calls 50] [--json out.json]
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]

import numpy as np  # noqa: E402
import torch  # noqa: E402

import art_planner_b200 as ap  # noqa: E402
from art_planner_b200 import build, costnet, synth  # noqa: E402


def gpu_info() -> str:
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv"],
                       capture_output=True, text=True, check=True)
    return r.stdout.strip()


def event_ms(fn, calls: int) -> float:
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    s.record()
    for _ in range(calls):
        fn()
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e) / calls


def host_ms(fn, calls: int) -> float:
    fn()
    t = time.perf_counter()
    for _ in range(calls):
        fn()
    return (time.perf_counter() - t) * 1e3 / calls


def measure(name: str, m, n_edges: int, calls: int) -> dict:
    chk = ap.StateValidityChecker(synth.PARAMS_YAML, device=0)
    chk.setMap(m)
    chk.updateHeightField()
    obj = ap.MotionCostObjective(chk)
    obj.setWeights(costnet.make_state_dict(seed=5))
    obj.updateFeatures()
    h = chk.handle
    s1, s2 = synth.make_edges(m, n_edges, seed=4, dmin=0.5, dmax=2.0)
    t1, t2 = torch.from_numpy(s1).cuda(), torch.from_numpy(s2).cuda()
    d = np.sqrt((s2[:, 0] - s1[:, 0]) ** 2 + (s2[:, 1] - s1[:, 1]) ** 2)
    total = int(((d / 0.5).astype(np.int64) + 1).sum())
    rows = torch.empty((total, 6), dtype=torch.float32, device="cuda")
    c3 = torch.empty((total, 3), dtype=torch.float32, device="cuda")
    cost = torch.empty(n_edges, dtype=torch.float64, device="cuda")
    # the offsets as the Python mirror builds them, outside the timed window
    off = torch.zeros(n_edges + 1, dtype=torch.int64, device="cuda")
    off[1:] = torch.cumsum((torch.sqrt((t2[:, 0] - t1[:, 0]) ** 2 + (t2[:, 1] - t1[:, 1]) ** 2) / 0.5).to(torch.int64) + 1, 0)
    off32 = off.to(torch.int32)
    assert int(off[-1].item()) == total
    lib = h.lib

    def split():
        h.check(lib.artp_motion_cost_split_device(h.h, C.c_void_p(t1.data_ptr()), C.c_void_p(t2.data_ptr()), n_edges,
                                                  C.c_void_p(off32.data_ptr()), total, C.c_void_p(rows.data_ptr()),
                                                  C.c_void_p(c3.data_ptr()), C.c_void_p(cost.data_ptr()),
                                                  C.c_void_p(torch.cuda.current_stream().cuda_stream)))

    def head():
        h.check(lib.artp_motion_cost_device(h.h, C.c_void_p(rows.data_ptr()), total, C.c_void_p(c3.data_ptr()),
                                            C.c_void_p(torch.cuda.current_stream().cuda_stream)))

    split_ms = event_ms(split, calls)
    head_ms = event_ms(head, calls)
    host_e2e_ms = host_ms(lambda: obj.motionCostBatch(s1, s2), max(5, calls // 4))
    # per-edge baselines over 2 000 edges
    k = 2000
    rows_np = rows.cpu().numpy()
    off_np = off.cpu().numpy()
    per_edge_split_ms = host_ms(lambda: [obj.motionCost(s1[i], s2[i]) for i in range(k)], 1)
    per_edge_query_ms = host_ms(lambda: [obj.getCost(obj.costQuery(rows_np[off_np[i]:off_np[i + 1]])) for i in range(k)], 1)
    # a 300-state path: one batch against 299 per-edge calls
    path = np.concatenate([s1[:1], s2[:299]])
    path_batch_ms = host_ms(lambda: obj.pathCost(path), 20)
    path_loop_ms = host_ms(lambda: [obj.motionCost(path[i], path[i + 1]) for i in range(299)], 3)
    return {
        "case": name, "edges": n_edges, "pieces": total,
        "split_device_ms": split_ms, "head_only_ms": head_ms, "rows_plus_reduce_ms": split_ms - head_ms,
        "split_device_edges_per_s": n_edges / split_ms * 1e3, "split_device_pieces_per_s": total / split_ms * 1e3,
        "host_e2e_ms": host_e2e_ms, "host_e2e_edges_per_s": n_edges / host_e2e_ms * 1e3,
        "per_edge_motionCost_edges_per_s": k / per_edge_split_ms * 1e3,
        "per_edge_costQuery_edges_per_s": k / per_edge_query_ms * 1e3,
        "path300_batch_us": path_batch_ms * 1e3, "path300_per_edge_us": path_loop_ms * 1e3,
    }


def main() -> None:
    ap_ = argparse.ArgumentParser()
    ap_.add_argument("--calls", type=int, default=50)
    ap_.add_argument("--edges", type=int, default=100_000)
    ap_.add_argument("--json", default=None)
    a = ap_.parse_args()
    assert torch.cuda.is_available(), "needs a CUDA device"
    assert a.calls >= 20
    build.build()
    info = gpu_info()
    print(info)
    import cases
    res = [measure("256x256 patch", cases.c4_map(), a.edges, a.calls),
           measure("1000x1000 map", synth.make_fbm_map(1000, 1000, 0.04, seed=2, amp=0.6), a.edges, a.calls)]
    for r in res:
        print(f"\n{r['case']}: {r['edges']} edges, {r['pieces']} pieces")
        print(f"  split device call      {r['split_device_ms']:.4f} ms  ({r['split_device_edges_per_s']:.3e} edges/s, "
              f"{r['split_device_pieces_per_s']:.3e} pieces/s)")
        print(f"  head alone, same rows  {r['head_only_ms']:.4f} ms  (rows + reduce add {r['rows_plus_reduce_ms']:.4f} ms, "
              f"{100 * r['rows_plus_reduce_ms'] / r['head_only_ms']:.1f} % of the head)")
        print(f"  host entry point e2e   {r['host_e2e_ms']:.3f} ms  ({r['host_e2e_edges_per_s']:.3e} edges/s)")
        print(f"  per-edge motionCost    {r['per_edge_motionCost_edges_per_s']:.3e} edges/s;  per-edge costQuery "
              f"{r['per_edge_costQuery_edges_per_s']:.3e} edges/s")
        print(f"  300-state pathCost     {r['path300_batch_us']:.1f} us as one batch, {r['path300_per_edge_us']:.1f} us as 299 calls")
    if a.json:
        with open(a.json, "w") as f:
            json.dump({"gpu": info, "results": res}, f, indent=1)


if __name__ == "__main__":
    main()
