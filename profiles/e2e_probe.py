"""e2e probe: host-buffer API throughput for 1M poses, plus raw H2D bandwidth."""
import os, sys, time
R = os.path.dirname(os.path.dirname(os.path.abspath(__file__))); sys.path.insert(0, R)
import numpy as np, torch
import art_planner_b200 as ap
from art_planner_b200 import synth
import bench
m, poses = bench.make_inputs(0, 1_000_000)
from art_planner_b200 import capi
B = [capi.HostBuffer((len(poses), 7), np.float64), capi.HostBuffer((len(poses), 7), np.float32), capi.HostBuffer((len(poses),), np.uint8)]
B[0].array[:] = poses; B[1].array[:] = poses.astype(np.float32)
hp, hp32, hv = (torch.from_numpy(b.array) for b in B)
if len(sys.argv) > 1 and sys.argv[1] == "bw":
    for mb in (7, 28, 56):
        n = mb << 20
        h = torch.empty(n, dtype=torch.uint8).pin_memory(); d = torch.empty(n, dtype=torch.uint8, device='cuda')
        for _ in range(3): d.copy_(h, non_blocking=True)
        torch.cuda.synchronize(); t = time.perf_counter()
        for _ in range(20): d.copy_(h, non_blocking=True)
        torch.cuda.synchronize(); dt = (time.perf_counter() - t) / 20
        print(f"H2D {mb} MiB pinned: {n/dt/1e9:.1f} GB/s")
chk = ap.StateValidityChecker(synth.PARAMS_YAML, device=0); chk.setMap(m); chk.updateHeightField()
for f32, h in ((True, hp32), (False, hp)):
    for _ in range(5): chk.isValidHostPtr(h.data_ptr(), len(poses), hv.data_ptr(), f32=f32)
    t = time.perf_counter()
    for _ in range(30): chk.isValidHostPtr(h.data_ptr(), len(poses), hv.data_ptr(), f32=f32)
    dt = (time.perf_counter() - t) / 30
    print(f"f32={f32}: {dt*1e3:.3f} ms  {len(poses)/dt/1e9:.3f} e9 poses/s")
