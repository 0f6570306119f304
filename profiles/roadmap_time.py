"""Time PRMMotionCost's sampleGraph at the shipped caps (10 000 vertices / 50 000 edges, recompute every 1000) on the
configs[1] map (1000 x 1000 fBm) at both roughness levels, three ways, and check that all three build the same roadmap:
  device       artp_roadmap_sample_graph: every milestone on the device, no host synchronisation between milestones
  host loop    the same loop driven from the host with this library: device candidates, host kNN, one
               artp_check_edge_interiors call per milestone, the distribution re-applied with updateDistribution
  reference    oracle/roadmap_oracle.py with isValid answered by the compiled reference's ODE, on the first PREFIX
               milestones (the whole run takes minutes), compared with the device roadmap's prefix
Prints one JSON line with the card's name and power limit."""
import dataclasses
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]

import numpy as np  # noqa: E402

import art_planner_b200 as ap  # noqa: E402
from art_planner_b200 import synth  # noqa: E402
from oracle import basic_oracle as bo  # noqa: E402
from oracle import orc  # noqa: E402
from oracle import roadmap_oracle as ro  # noqa: E402
from oracle import sample_distribution_oracle as sdo  # noqa: E402

CAPS = (10000, 50000, 1000)
PREFIX = 60


def host_loop(chk, smp, caps, dp_on=True):
    """sampleGraph driven from the host: returns (roadmap, draws used)."""
    mv = ap.MotionValidator(chk)
    rm = ro.Roadmap()
    draw, n_proc, chunk = 0, 0, 4096
    while rm.V < caps[0] and rm.E < caps[1]:
        while True:
            cand = smp.sampleUniformBatch(chunk, first=draw)
            ok = ~np.isnan(cand[:, 0])
            v = np.zeros(chunk, bool)
            v[ok] = chk.isValidBatch(cand[ok]).astype(bool)
            hit = np.flatnonzero(v)
            if hit.size:
                break
            draw += chunk
        s = cand[hit[0]]
        draw += int(hit[0]) + 1
        V = rm.V
        nbrs = ro.nearest(s, rm.states[:V], min(ro.k_star(V + 1), V))
        S = rm.states[:V].copy()
        m = rm._vertex(s, ro.MILESTONE)
        if len(nbrs):
            prefix, n_interp = mv.checkEdgeInteriors(np.repeat(s[None], len(nbrs), 0), S[nbrs])
            for n, p, ni in zip(nbrs, prefix, n_interp):
                if ni == 0:
                    rm._edge(m, int(n))
                    continue
                prev, div = m, 1.0 / (int(ni) + 1)
                for step in range(1, int(p) + 1):
                    w = rm._vertex(ro.interpolate(s, S[n], step * div), ro.INTERPOLATED)
                    rm._edge(prev, w)
                    prev = w
                if p == ni:
                    rm._edge(prev, int(n))
        if dp_on and rm.V // caps[2] > n_proc:
            smp.updateDistribution(rm.density_states())
            n_proc += 1
    return rm, draw


def run(level):
    m = synth.make_fbm_map(1000, 1000) if level == "gentle" else \
        synth.make_fbm_map(1000, 1000, amp=1.2, wavelength=3.0, persistence=0.7)
    rp = synth.PARAMS_YAML
    trav, obs = synth.make_traversability(m, seed=13)
    _, thr = bo.masked_elevation(m.elevation, trav, obs, m.res, bo.BasicParams())
    chk = ap.StateValidityChecker(rp, device=0)
    chk.setMap(m)
    chk.updateHeightField()
    chk.setSampleFilter(thr, obs)
    L = synth.make_sampler_layers(m, seed=7)
    sp = dataclasses.replace(synth.sampler_params_for(m), use_inverse_vertex_density=True, use_max_prob_unknown_samples=True)
    times = []
    for _ in range(4):
        smp = ap.SE3FromSE2Sampler(chk, L, sp, seed=1234)
        rm = ap.PRMRoadmap(chk, 20000, 60000)
        t0 = time.perf_counter()
        used = rm.sampleGraph(smp, *CAPS)          # returns after the call's stream synchronise
        times.append((time.perf_counter() - t0) * 1e3)
    st, kinds = rm.vertices()
    edges = rm.edges()
    n_ms = int((kinds == ro.MILESTONE).sum())
    dev = float(np.median(times[1:]))
    # the host-driven loop on a fresh sampler over the same stream and layers
    smp = ap.SE3FromSE2Sampler(chk, L, sp, seed=1234)
    t0 = time.perf_counter()
    hrm, h_used = host_loop(chk, smp, CAPS)
    host_ms = (time.perf_counter() - t0) * 1e3
    hst, hkinds, hedges = hrm.result()
    same_host = h_used == used and np.array_equal(hkinds, kinds) and np.array_equal(hedges, edges) and \
        float(np.abs(hst - st).max()) <= 1e-9
    assert same_host, "the host-driven loop built another roadmap"
    out = {"vertices": int(len(kinds)), "edges": int(len(edges)), "milestones": n_ms, "draws_used": int(used),
           "device_ms": dev, "device_milestones_per_s": n_ms / dev * 1e3,
           "host_loop_ms": host_ms, "host_loop_milestones_per_s": n_ms / host_ms * 1e3, "host_equal": bool(same_host)}
    if orc.available("reference"):
        o = orc.Oracle(rp, "reference")
        o.set_map(m)
        ref = ro.Roadmap()
        t0 = time.perf_counter()
        ro.sample_graph(ref, o, m, L, sp, rp.reach_z, 1234, 0, *CAPS, 1 << 26,
                        sdo.DistributionParams(True, (rp.torso_length + rp.torso_width) * 0.25, True, 0.1),
                        sdo.sample_filter(thr, rp, m.res), obs, max_milestones=PREFIX)
        cpu_ms = (time.perf_counter() - t0) * 1e3
        rst, rkinds, redges = ref.result()
        same_ref = np.array_equal(rkinds, kinds[:ref.V]) and np.array_equal(redges, edges[:ref.E]) and \
            float(np.abs(rst - st[:ref.V]).max()) <= 1e-9
        assert same_ref, "the compiled-reference restatement built another roadmap prefix"
        out.update({"reference_prefix_milestones": PREFIX, "reference_prefix_vertices": int(ref.V), "reference_cpu_ms": cpu_ms,
                    "reference_milestones_per_s": PREFIX / cpu_ms * 1e3, "reference_equal": bool(same_ref)})
    else:
        out["reference"] = "not measured (oracle/_ref not built)"
    return out


def main():
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip()
    out = {"gpu": gpu, "caps": CAPS, "gentle": run("gentle"), "rough": run("rough")}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
