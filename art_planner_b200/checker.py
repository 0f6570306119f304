"""Host-side mirror of the reference's plugin interface for the hot path, over the C ABI (include/artp.h).

Names, argument meaning and error behaviour follow the reference:
  StateValidityChecker   art_planner/include/art_planner/validity_checker/validity_checker.h:21-39
                         (setMap / updateHeightField / hasMap / isValid); installed by Planner
                         (art_planner/src/planner.cpp:125-127,162)
  MotionValidator        ompl::base::MotionValidator::checkMotion as used at
                         art_planner/src/planners/prm_motion_cost.cpp:652 (OMPL DiscreteMotionValidator)
  PathLengthObjective    art_planner/src/objectives/path_length_objective.cpp:26-70
A state is 7 doubles (x y z qx qy qz qw), the SE3StateSpace::StateType fields the reference reads
(art_planner/include/art_planner/utils.h:25-38). Batches are [n, 7] float64 arrays; numpy arrays go through
the host-buffer entry points (H2D/D2H inside), CUDA torch tensors through the *_device entry points on
torch's current stream.
"""
from __future__ import annotations

import ctypes as C

import numpy as np

from . import capi


def _is_torch_cuda(x) -> bool:
    return hasattr(x, "is_cuda") and bool(x.is_cuda)


class _Handle:
    """Owns one artp_handle (one CUDA device)."""

    def __init__(self, robot_params, device: int = 0, cost_weights=(0.0, 1.0, 5.0), risk_threshold=0.5):
        self.lib = capi.load()
        self.params = robot_params
        self.device = device
        p = capi.make_params(robot_params, device, cost_weights, risk_threshold)
        h = C.c_void_p()
        rc = self.lib.artp_create(C.byref(p), C.byref(h))
        if rc != 0:
            raise capi.ArtpError(rc, self.lib.artp_last_error(None).decode())
        self.h = h

    def check(self, rc: int) -> None:
        if rc != 0:
            raise capi.ArtpError(rc, self.lib.artp_last_error(self.h).decode())

    def close(self) -> None:
        if getattr(self, "h", None):
            self.lib.artp_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def stats(self) -> dict:
        s = capi.ArtpStats()
        self.check(self.lib.artp_get_stats(self.h, C.byref(s)))
        return {k: int(getattr(s, k)) for k, _ in capi.ArtpStats._fields_}


def _stream_ptr():
    import torch
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _column_major_cuda(layer, what: str):
    """(rows, cols) of a column-major float32 CUDA layer (a transposed contiguous cols x rows tensor)."""
    import torch
    if layer.dtype != torch.float32 or not layer.t().is_contiguous():
        raise ValueError(f"{what}: a CUDA layer must be float32 and column-major (a transposed contiguous tensor)")
    return layer.shape


class StateValidityChecker:
    """art_planner::StateValidityChecker on the GPU (validity_checker.cpp:9-45)."""

    def __init__(self, params, device: int = 0, handle: _Handle | None = None):
        self._h = handle or _Handle(params, device)
        self._map = None

    # -- reference interface ------------------------------------------------------------------
    def setMap(self, synth_map) -> None:             # validity_checker.cpp:20-23
        self._map = synth_map

    def updateHeightField(self, window=None) -> None:   # validity_checker.cpp:27-31 -> setHeightField
        """window = (row0, nrows): upload only that row slab of the map (spatial shard, artp_set_map_window); geometry stays
        that of the full map, so verdicts are identical to a checker holding everything."""
        if self._map is None:
            raise capi.ArtpError(capi.ARTP_E_NOMAP, "setMap() was not called")
        m = self._map
        if window is not None:
            row0, nrows = int(window[0]), int(window[1])
            e = np.asfortranarray(m.elevation[row0:row0 + nrows, :], dtype=np.float32)
            k = np.asfortranarray(m.elevation_masked[row0:row0 + nrows, :], dtype=np.float32)
            self._h.check(self._h.lib.artp_set_map_window(self._h.h, e.ctypes.data, k.ctypes.data, m.elevation.shape[0],
                                                          m.elevation.shape[1], float(m.res), float(m.cx), float(m.cy), row0, nrows))
            return
        e = np.asfortranarray(m.elevation, dtype=np.float32)
        k = np.asfortranarray(m.elevation_masked, dtype=np.float32)
        if e.shape != k.shape:
            raise capi.ArtpError(capi.ARTP_E_INVALID, "layer shapes differ")
        self._h.check(self._h.lib.artp_set_map(self._h.h, e.ctypes.data, k.ctypes.data, e.shape[0], e.shape[1],
                                               float(m.res), float(m.cx), float(m.cy)))

    def hasMap(self) -> bool:                        # validity_checker.cpp:33-35
        return bool(self._h.lib.artp_has_map(self._h.h))

    def isValid(self, state) -> bool:                # validity_checker.cpp:39-45 (batch of 1: latency path)
        s = np.ascontiguousarray(state, dtype=np.float64).reshape(1, 7)
        return bool(self.isValidBatch(s)[0])

    # -- batched entry points -----------------------------------------------------------------
    def isValidBatch(self, states, out=None):
        """states [n, 7] float64 (numpy or CUDA torch tensor) -> uint8 mask of the same kind."""
        lib, h = self._h.lib, self._h
        if _is_torch_cuda(states):
            import torch
            assert states.dtype in (torch.float64, torch.float32) and states.is_contiguous() and states.shape[-1] == 7
            n = states.shape[0]
            if out is None:
                out = torch.empty(n, dtype=torch.uint8, device=states.device)
            fn = lib.artp_check_poses_device if states.dtype == torch.float64 else lib.artp_check_poses_f32_device
            h.check(fn(h.h, C.c_void_p(states.data_ptr()), n, C.c_void_p(out.data_ptr()), _stream_ptr()))
            return out
        f32 = getattr(states, "dtype", None) == np.float32
        s = np.ascontiguousarray(states, dtype=np.float32 if f32 else np.float64)
        assert s.ndim == 2 and s.shape[1] == 7
        n = s.shape[0]
        if out is None:
            out = np.empty(n, dtype=np.uint8)
        fn = lib.artp_check_poses_f32 if f32 else lib.artp_check_poses
        h.check(fn(h.h, s.ctypes.data, n, out.ctypes.data))
        return out

    def sampleValidBatch(self, sampler, n_wanted: int, batch: int = 65536, max_draws: int = 1 << 24):
        """The rejection-sampling loop `do sampleUniform(s) while (!isValid(s))` (prm_motion_cost.cpp:171-194,
        lazy_prm_star_min_update.cpp:549-556) in batches: sampler(m) -> [m, 7] candidates; valid ones are kept in draw
        order until n_wanted states are collected or max_draws candidates were drawn. Returns (states, drawn)."""
        kept, have, drawn = [], 0, 0
        while have < n_wanted and drawn < max_draws:
            m = min(batch, max_draws - drawn)
            cand = np.ascontiguousarray(sampler(m))
            drawn += m
            ok = cand[self.isValidBatch(cand) != 0][: n_wanted - have]
            kept.append(ok)
            have += len(ok)
        return (np.concatenate(kept) if kept else np.zeros((0, 7))), drawn

    def isValidHostPtr(self, states_ptr: int, n: int, valid_ptr: int, f32: bool = False) -> None:
        """Raw host pointers (e.g. pinned torch tensors): the exact call an OMPL adapter makes. f32: the states were
        already cast to float (what Pose3FromSE3 does first) -- identical results, half the H2D bytes."""
        fn = self._h.lib.artp_check_poses_f32 if f32 else self._h.lib.artp_check_poses
        self._h.check(fn(self._h.h, C.c_void_p(states_ptr), n, C.c_void_p(valid_ptr)))

    def compactValid(self, valid, base: int = 0):
        """Ordered indices (int64, base + i) of the non-zero entries of a CUDA uint8 mask; returns (indices, count)
        as CUDA tensors -- the payload of the multi-GPU index all-gather."""
        import torch
        n = valid.shape[0]
        idx = torch.empty(n, dtype=torch.int64, device=valid.device)
        cnt = torch.zeros(1, dtype=torch.int32, device=valid.device)
        self._h.check(self._h.lib.artp_compact_valid_device(self._h.h, C.c_void_p(valid.data_ptr()), n, int(base),
                                                            C.c_void_p(idx.data_ptr()), C.c_void_p(cnt.data_ptr()),
                                                            _stream_ptr()))
        return idx, cnt

    def processBasic(self, elevation, traversability, observed, res: float, bp):
        """processors::Basic::setMaskedElevationAndTraversability (basic.cpp:42-106) on the device, after the inpainting:
        returns (elevation_masked, traversability_thresholded), float32 Fortran-order. bp: an object with the fields of
        artp_basic_params (oracle.basic_oracle.BasicParams has them)."""
        e = np.asfortranarray(elevation, dtype=np.float32)
        t = np.asfortranarray(traversability, dtype=np.float32)
        o = None if observed is None else np.asfortranarray(observed, dtype=np.float32)
        p = capi.basic_params(bp)
        masked = np.empty(e.shape, np.float32, order="F"); thr = np.empty(e.shape, np.float32, order="F")
        self._h.check(self._h.lib.artp_process_basic(self._h.h, e.ctypes.data, t.ctypes.data, None if o is None else o.ctypes.data,
                                                     e.shape[0], e.shape[1], float(res), C.byref(p), masked.ctypes.data, thr.ctypes.data))
        return masked, thr

    def estimateNormals(self, estimation_radius: float, want_host: bool = True):
        """art_planner::estimateNormals (utils.cpp:213-324) for the current elevation layer, on the device; the layers
        stay resident as the sampler's inputs. Returns (normal_x, normal_y, normal_z, plane_fit_std_dev) float32
        Fortran-order arrays, or None when want_host is False."""
        rows, cols = self._map.elevation.shape
        outs = [np.empty((rows, cols), np.float32, order="F") for _ in range(4)] if want_host else [None] * 4
        self._h.check(self._h.lib.artp_estimate_normals(self._h.h, float(estimation_radius),
                                                        *[None if a is None else a.ctypes.data for a in outs]))
        return tuple(outs) if want_host else None

    def computeSampleCdf(self, sample_probability, want_host: bool = True):
        """computeCumulativeProbabilityDistribution (probability_distribution.cpp:20-46) on the device; the CDF layers stay
        resident for SE3FromSE2Sampler. Returns (cum_prob [rows, cols] F-order, cum_prob_rowwise [rows]) or None."""
        p = np.asfortranarray(sample_probability, dtype=np.float32)
        cum = np.empty(p.shape, np.float32, order="F") if want_host else None
        row = np.empty(p.shape[0], np.float32) if want_host else None
        self._h.check(self._h.lib.artp_compute_sample_cdf(self._h.h, p.ctypes.data, None if cum is None else cum.ctypes.data,
                                                          None if row is None else row.ctypes.data))
        return (cum, row) if want_host else None

    def setSampleFilter(self, traversability_thresholded=None, observed=None, want_host: bool = True):
        """Basic::setTraversabilityFilter (basic.cpp:110-125) on the device for the current map, with the "observed" layer the
        unknown-space cap reads; both stay resident for updateSampleDistribution. None: the layer the last processBasic on
        this checker received (observed) / produced (traversability_thresholded). Returns traversability_sample_filter
        (float32 F-order) or None."""
        rows, cols = self._map.elevation.shape
        f = lambda a: None if a is None else np.asfortranarray(a, dtype=np.float32)
        t, o = f(traversability_thresholded), f(observed)
        for a in (t, o):
            if a is not None and a.shape != (rows, cols):
                raise capi.ArtpError(capi.ARTP_E_INVALID, "layer shape differs from the map's")
        out = np.empty((rows, cols), np.float32, order="F") if want_host else None
        self._h.check(self._h.lib.artp_set_sample_filter(self._h.h, *[None if a is None else a.ctypes.data for a in (t, o, out)]))
        return out

    def updateSampleDistribution(self, vertex_states, dp, want_host: bool = True):
        """computeInverseSampleDensity -> applyBaseSampleDistribution -> applyMaxUnknownProbability ->
        computeCumulativeProbabilityDistribution (planner.cpp:39-58) on the device for the roadmap's vertex states [n, 7]
        (only x, y read). dp: an object with the fields of artp_sample_distribution_params. The CDF stays resident: re-arm
        the sampler afterwards (SE3FromSE2Sampler.updateDistribution does both). A CUDA float64 tensor goes through the
        device entry point on the current stream and returns None; else returns (sample_probability, cum_prob,
        cum_prob_rowwise) when want_host."""
        lib, h = self._h.lib, self._h
        p = capi.ArtpSampleDistributionParams(int(dp.use_inverse_vertex_density), float(dp.density_blur_radius),
                                              int(dp.use_max_prob_unknown_samples), float(dp.max_prob_unknown_samples))
        if _is_torch_cuda(vertex_states):
            import torch
            assert vertex_states.dtype == torch.float64 and vertex_states.is_contiguous() and vertex_states.shape[-1] == 7
            h.check(lib.artp_update_sample_distribution_device(h.h, C.byref(p), C.c_void_p(vertex_states.data_ptr()),
                                                               vertex_states.shape[0], _stream_ptr()))
            return None
        v = np.ascontiguousarray(vertex_states, dtype=np.float64).reshape(-1, 7)
        rows, cols = self._map.elevation.shape
        outs = [np.empty((rows, cols), np.float32, order="F"), np.empty((rows, cols), np.float32, order="F"),
                np.empty(rows, np.float32)] if want_host else [None] * 3
        h.check(lib.artp_update_sample_distribution(h.h, C.byref(p), v.ctypes.data, v.shape[0],
                                                    *[None if a is None else a.ctypes.data for a in outs]))
        return tuple(outs) if want_host else None

    def findValidNear(self, centres, radius, n_iter: int, offsets=None, seed: int = 0, first_draw: int = 0):
        """StartState / GoalStateRegion::sampleGoal (start.cpp:7-41, goal.cpp:11-41) for n queries in one call: the first
        valid of the centre and the centre moved in x / y by offsets 1..n_iter; none valid -> the last candidate. centres
        [n, 7] float64, radius scalar or [n], offsets [n, n_iter, 2] or None (the Philox "ARTB" stream from first_draw,
        see artp.h). Returns (states [n, 7], index int32 [n]: candidate k, or -1). CUDA float64 tensors go through the
        device entry point on the current stream (radius and offsets then CUDA tensors too)."""
        lib, h = self._h.lib, self._h
        if not 0 <= int(n_iter) < 2 ** 32:
            raise capi.ArtpError(capi.ARTP_E_INVALID, "n_iter must lie in [0, 2^32)")
        if _is_torch_cuda(centres):
            import torch
            assert centres.dtype == torch.float64 and centres.is_contiguous() and centres.shape[-1] == 7
            n = centres.shape[0]
            r = torch.as_tensor(radius, dtype=torch.float64, device=centres.device).expand(n).contiguous()
            off = None if offsets is None else offsets.contiguous()
            assert off is None or (off.dtype == torch.float64 and off.numel() == n * int(n_iter) * 2)
            out = torch.empty((n, 7), dtype=torch.float64, device=centres.device)
            idx = torch.empty(n, dtype=torch.int32, device=centres.device)
            h.check(lib.artp_find_valid_near_device(h.h, C.c_void_p(centres.data_ptr()), n, C.c_void_p(r.data_ptr()), int(n_iter),
                                                    None if off is None else C.c_void_p(off.data_ptr()), int(seed), int(first_draw),
                                                    C.c_void_p(out.data_ptr()), C.c_void_p(idx.data_ptr()), _stream_ptr()))
            return out, idx
        c = np.ascontiguousarray(centres, dtype=np.float64).reshape(-1, 7)
        n = c.shape[0]
        r = np.ascontiguousarray(np.broadcast_to(np.asarray(radius, dtype=np.float64), (n,)))
        off = None
        if offsets is not None:
            off = np.ascontiguousarray(offsets, dtype=np.float64)
            assert off.size == n * int(n_iter) * 2
        out = np.empty((n, 7), np.float64)
        idx = np.empty(n, np.int32)
        h.check(lib.artp_find_valid_near(h.h, c.ctypes.data, n, r.ctypes.data, int(n_iter), None if off is None else off.ctypes.data,
                                         int(seed), int(first_draw), out.ctypes.data, idx.ctypes.data))
        return out, idx

    def ballOffsets(self, seed: int, first_draw: int, n: int, n_iter: int, radius):
        """The [n, n_iter, 2] offsets findValidNear draws from its stream (offsets=None) for the same seed / first_draw."""
        lib, h = self._h.lib, self._h
        r = np.ascontiguousarray(np.broadcast_to(np.asarray(radius, dtype=np.float64), (n,)))
        out = np.empty((n, int(n_iter), 2), np.float64)
        h.check(lib.artp_ball_offsets(h.h, int(seed), int(first_draw), n, int(n_iter), r.ctypes.data, out.ctypes.data))
        return out

    def poseFrom2D(self, states):
        """The goal projection of Planner::plan (planner.cpp:223-237, Map::get3DPoseFrom2D map.cpp:77-90) on the device:
        states [n, 7] -> (states [n, 7], inside uint8 [n]); states off the map come back unchanged with inside == 0.
        Needs the current map's normals (estimateNormals, or a sampler set with host normal layers)."""
        s = np.ascontiguousarray(states, dtype=np.float64).reshape(-1, 7)
        out = np.empty_like(s)
        inside = np.empty(s.shape[0], np.uint8)
        self._h.check(self._h.lib.artp_pose_from_2d(self._h.h, s.ctypes.data, s.shape[0], out.ctypes.data, inside.ctypes.data))
        return out, inside

    def isValidBatchBits(self, states, out_valid, out_bits):
        """One shard step of the multi-GPU path: verdict bytes + bit-packed mask (CUDA float64 states), one call."""
        n = states.shape[0]
        self._h.check(self._h.lib.artp_check_poses_bits_device(self._h.h, C.c_void_p(states.data_ptr()), n,
                                                               C.c_void_p(out_valid.data_ptr()), C.c_void_p(out_bits.data_ptr()),
                                                               _stream_ptr()))

    def compactValidU32(self, valid, base: int = 0, out_idx=None, out_cnt=None):
        """Ordered 32-bit indices (base + i) of the non-zero entries of a CUDA uint8 mask -> (indices int32 view, count)."""
        import torch
        n = valid.shape[0]
        if out_idx is None:
            out_idx = torch.empty(n, dtype=torch.int32, device=valid.device)
        if out_cnt is None:
            out_cnt = torch.zeros(1, dtype=torch.int32, device=valid.device)
        self._h.check(self._h.lib.artp_compact_valid_u32_device(self._h.h, C.c_void_p(valid.data_ptr()), n, int(base),
                                                                C.c_void_p(out_idx.data_ptr()), C.c_void_p(out_cnt.data_ptr()),
                                                                _stream_ptr()))
        return out_idx, out_cnt

    def packValidBits(self, valid, out=None):
        """CUDA uint8 mask [n] -> bit-packed int32 words [(n+31)//32] (item i = bit i&31 of word i>>5)."""
        import torch
        n = valid.shape[0]
        if out is None:
            out = torch.empty((n + 31) // 32, dtype=torch.int32, device=valid.device)
        self._h.check(self._h.lib.artp_pack_valid_bits_device(self._h.h, C.c_void_p(valid.data_ptr()), n,
                                                              C.c_void_p(out.data_ptr()), _stream_ptr()))
        return out

    def compactBits(self, bits, n: int, base: int = 0, out_idx=None, out_cnt=None):
        """Ordered indices of the set bits among the first n of a bit-packed CUDA mask -> (indices int64 [n], count)."""
        import torch
        if out_idx is None:
            out_idx = torch.empty(n, dtype=torch.int64, device=bits.device)
        if out_cnt is None:
            out_cnt = torch.empty(1, dtype=torch.int32, device=bits.device)
        self._h.check(self._h.lib.artp_compact_bits_device(self._h.h, C.c_void_p(bits.data_ptr()), n, int(base),
                                                           C.c_void_p(out_idx.data_ptr()), C.c_void_p(out_cnt.data_ptr()),
                                                           _stream_ptr()))
        return out_idx, out_cnt

    def setMode(self, mode: int) -> None:
        self._h.check(self._h.lib.artp_set_mode(self._h.h, int(mode)))

    def pollError(self) -> None:
        """Raise ArtpError(ARTP_E_LIMIT) if an asynchronous (device-buffer) call hit the plane-grouping overflow since the
        last poll (the affected poses were reported invalid). Synchronise the stream first."""
        self._h.check(self._h.lib.artp_poll_error(self._h.h))

    def inpaint(self, layer):
        """inpaintMatrix (art_planner/src/utils.cpp:13-63) of a rows x cols grid_map layer (NaN = unknown) on the device:
        artp_inpaint_layer for a numpy array (returns a column-major float32 array), artp_inpaint_layer_device for a CUDA
        tensor (column-major: a transposed contiguous cols x rows float32 tensor; returns the same layout, on the current
        stream)."""
        if _is_torch_cuda(layer):
            import torch
            rows, cols = layer.shape
            if layer.dtype != torch.float32 or not layer.t().is_contiguous():
                raise ValueError("inpaint: a CUDA layer must be float32 and column-major (a transposed contiguous tensor)")
            out = torch.empty((cols, rows), dtype=torch.float32, device=layer.device).t()
            self._h.check(self._h.lib.artp_inpaint_layer_device(self._h.h, layer.data_ptr(), rows, cols, out.data_ptr(),
                                                                _stream_ptr()))
            return out
        a = np.asfortranarray(layer, dtype=np.float32)
        out = np.empty(a.shape, np.float32, order="F")
        self._h.check(self._h.lib.artp_inpaint_layer(self._h.h, a.ctypes.data, a.shape[0], a.shape[1], out.ctypes.data))
        return out

    def debugSetGroupCapacity(self, max_triangles: int) -> None:
        self._h.check(self._h.lib.artp_debug_set_group_capacity(self._h.h, int(max_triangles)))

    def debugReachQueue(self):
        """Records of the one-warp-per-box reach queue of the last call's last round: (zone [n, 4] int32 x0, x1, z0, z1;
        flags [n] uint32), read from the device (BoxRec, artp_kernels.cuh)."""
        import numpy as np
        n = C.c_size_t(0)
        self._h.check(self._h.lib.artp_debug_get_reach_queue(self._h.h, None, 0, C.byref(n)))
        buf = np.empty((n.value, 20), dtype=np.uint32)
        self._h.check(self._h.lib.artp_debug_get_reach_queue(self._h.h, C.c_void_p(buf.ctypes.data), n.value, C.byref(n)))
        return buf[:, 14:18].view(np.int32).copy(), buf[:, 19].copy()

    def stats(self) -> dict:
        return self._h.stats()

    def setTiming(self, enable: bool) -> None:
        self._h.check(self._h.lib.artp_set_timing(self._h.h, int(bool(enable))))

    def lastKernelTimesMs(self):
        """(classify ms, box warp stage ms, plane-grouping stage ms) of the most recent check call (CUDA events
        recorded by the library on the call's stream)."""
        ms = (C.c_float * 3)()
        self._h.check(self._h.lib.artp_get_last_timing(self._h.h, ms))
        return float(ms[0]), float(ms[1]), float(ms[2])

    def lastStageTimesMs(self):
        """(classify, big-tile queue, reach queue (warp per box), reach queue (8-lane groups), plane grouping) ms of the most recent
        check call."""
        ms = (C.c_float * 5)()
        self._h.check(self._h.lib.artp_get_last_stage_timing(self._h.h, ms))
        return tuple(float(x) for x in ms)

    @property
    def handle(self) -> _Handle:
        return self._h


def _distribution_params(sp, rp) -> capi.ArtpSampleDistributionParams:
    """The distribution parameters from the sampler parameters `sp` and the robot's `rp`, with the reference Planner's
    density blur radius (planner.cpp:48)."""
    return capi.ArtpSampleDistributionParams(int(sp.use_inverse_vertex_density), (rp.torso_length + rp.torso_width) * 0.25,
                                             int(sp.use_max_prob_unknown_samples), float(sp.max_prob_unknown_samples))


class SE3FromSE2Sampler:
    """art_planner::SE3FromSE2Sampler::sampleUniform (src/sampler.cpp:82-131) on the device, plus the fused
    sample -> isValid -> compact form of the rejection loops around it (prm_motion_cost.cpp:171-194).

    `layers` carries normal_x/y/z, plane_fit_std_dev, cum_prob, cum_prob_rowwise (grid_map matrices);
    `sp` the sampler parameters (max_roll_pert, max_pitch_pert, sample_from_distribution, low, high).
    Must be re-created / setLayers() again after every setMap on the checker."""

    def __init__(self, checker: StateValidityChecker, layers, sp, seed: int = 0):
        self._c = checker
        self.seed = int(seed)
        self._next = 0
        self.setLayers(layers, sp)

    def setLayers(self, layers, sp) -> None:
        h, lib = self._c.handle, self._c.handle.lib
        f = lambda a: None if a is None else np.asfortranarray(a, dtype=np.float32)
        keep = [f(getattr(layers, "normal_x", None)), f(getattr(layers, "normal_y", None)),
                f(getattr(layers, "normal_z", None)), f(getattr(layers, "plane_fit_std_dev", None)),
                f(getattr(layers, "cum_prob", None)),
                None if getattr(layers, "cum_prob_rowwise", None) is None
                else np.ascontiguousarray(layers.cum_prob_rowwise, dtype=np.float32)]
        p = capi.ArtpSamplerParams(float(sp.max_roll_pert), float(sp.max_pitch_pert), int(sp.sample_from_distribution),
                                   (C.c_double * 2)(*sp.low), (C.c_double * 2)(*sp.high))
        h.check(lib.artp_set_sampler(h.h, C.byref(p), *[None if a is None else a.ctypes.data for a in keep]))
        self._sp, self._params, self._normals = sp, p, keep[:4]

    def updateDistribution(self, vertex_states) -> None:
        """The reApplyPreprocessing step of PRMMotionCostMaintainer::sampleGraph (prm_motion_cost.cpp:190-193): the sampling
        distribution from the roadmap's vertex states (with the filter / observed layers of the checker's setSampleFilter),
        then the sampler re-armed on the new device CDF. Parameters from `sp` (use_inverse_vertex_density,
        use_max_prob_unknown_samples, max_prob_unknown_samples) and the blur radius of planner.cpp:48."""
        h, lib = self._c.handle, self._c.handle.lib
        self._c.updateSampleDistribution(vertex_states, _distribution_params(self._sp, h.params), want_host=False)
        h.check(lib.artp_set_sampler(h.h, C.byref(self._params), *[None if a is None else a.ctypes.data for a in self._normals],
                                     None, None))

    def uniforms(self, first: int, n: int) -> np.ndarray:
        """The [n, 6] uniform01 variates of samples first..first+n-1 of this sampler's Philox stream."""
        h, lib = self._c.handle, self._c.handle.lib
        u = np.empty((n, 6), np.float64)
        h.check(lib.artp_sampler_uniforms(h.h, self.seed, int(first), n, u.ctypes.data))
        return u

    def sampleUniformBatch(self, n: int, u=None, first=None, want_cells: bool = False):
        """n candidates [n, 7]. u: optional [n, 6] variates (else the Philox stream from `first`, default: continue)."""
        h, lib = self._c.handle, self._c.handle.lib
        if first is None:
            first = self._next
            if u is None:
                self._next += n
        states = np.empty((n, 7), np.float64)
        rc = np.empty((n, 2), np.int32) if want_cells else None
        uu = None if u is None else np.ascontiguousarray(u, dtype=np.float64)
        assert uu is None or uu.shape == (n, 6)
        h.check(lib.artp_sample_states(h.h, None if uu is None else uu.ctypes.data, self.seed, int(first), n,
                                       states.ctypes.data, None if rc is None else rc.ctypes.data))
        return (states, rc) if want_cells else states

    def sampleUniform(self) -> np.ndarray:
        """One state, never NaN: in uniform mode a draw outside the map is redrawn from the next counter of the stream,
        like samplePositionInMap's loop (sampler.cpp:46-50)."""
        while True:
            s = self.sampleUniformBatch(1)[0]
            if not np.isnan(s[0]):
                return s

    def sampleUniformInside(self, n: int) -> np.ndarray:
        """n states, none NaN, in draw order (rejected outside-map candidates of the uniform mode are redrawn)."""
        out = []
        have = 0
        while have < n:
            s = self.sampleUniformBatch(n - have)
            s = s[~np.isnan(s[:, 0])]
            out.append(s)
            have += len(s)
        return np.concatenate(out) if out else np.zeros((0, 7))

    def sampleValidBatch(self, n_draw: int, first=None, capacity=None, out=None):
        """Draw n_draw candidates on the device, check them, return (valid states in draw order, n_valid).
        out: optional reusable [cap, 7] float64 host buffer (numpy array or pinned CPU torch tensor); a fresh
        58 MB numpy array per 2^20 draws costs more in page faults than the whole GPU pass."""
        h, lib = self._c.handle, self._c.handle.lib
        if first is None:
            first = self._next
            self._next += n_draw
        if out is None:
            cap = n_draw if capacity is None else int(capacity)
            out = np.empty((cap, 7), np.float64)
        else:
            cap = out.shape[0] if capacity is None else min(int(capacity), out.shape[0])
        ptr = out.ctypes.data if isinstance(out, np.ndarray) else out.data_ptr()
        nv = C.c_size_t(0)
        h.check(lib.artp_sample_valid(h.h, self.seed, int(first), n_draw, C.c_void_p(ptr), cap, C.byref(nv)))
        return out[: min(nv.value, cap)], nv.value

    def sampleValidDevice(self, n_draw: int, first: int, out, count):
        """Device buffers: out = CUDA float64 [cap, 7], count = CUDA int32 [1]; asynchronous on the current stream."""
        h, lib = self._c.handle, self._c.handle.lib
        h.check(lib.artp_sample_valid_device(h.h, self.seed, int(first), n_draw, C.c_void_p(out.data_ptr()), out.shape[0],
                                             C.c_void_p(count.data_ptr()), _stream_ptr()))


class PRMRoadmap:
    """PRMMotionCost's roadmap built on the device (prm_motion_cost.cpp:145-219, 236-247, 325-390): addValidMilestone with
    KStarStrategy's k nearest, the interior states of every connection at <= 0.5 m lateral spacing, and the valid prefixes
    as chains of vertices and edges. vertices() / edges() copy the store out in the order the reference's Boost graph
    numbers them. updateEdges() prices the edges in place with the loaded motion-cost network, solve() answers a query
    on the device, edgeCosts() copies the weights and flags out."""

    EDGE_VALID, EDGE_REMOVED = capi.ARTP_ROADMAP_EDGE_VALID, capi.ARTP_ROADMAP_EDGE_REMOVED
    SOLVED, NOT_CONNECTED, NO_FEASIBLE_PATH = capi.ARTP_SOLVE_SOLVED, capi.ARTP_SOLVE_NOT_CONNECTED, capi.ARTP_SOLVE_NO_FEASIBLE_PATH
    INVALID_START, INVALID_GOAL = capi.ARTP_SOLVE_INVALID_START, capi.ARTP_SOLVE_INVALID_GOAL

    MILESTONE, INTERPOLATED, QUERY = capi.ARTP_ROADMAP_MILESTONE, capi.ARTP_ROADMAP_INTERPOLATED, capi.ARTP_ROADMAP_QUERY

    def __init__(self, checker: StateValidityChecker, vertex_capacity: int = 60000, edge_capacity: int = 60000):
        self._c = checker
        self.vertex_capacity, self.edge_capacity = int(vertex_capacity), int(edge_capacity)
        self.clear()

    def clear(self) -> None:                             # PRMMotionCost::clear (:236-247)
        h = self._c.handle
        h.check(h.lib.artp_roadmap_clear(h.h, self.vertex_capacity, self.edge_capacity))

    def addValidMilestones(self, states) -> None:
        """addValidMilestone for each state in order: baseSolve's start / goal milestones (:451-479)."""
        h = self._c.handle
        s = np.ascontiguousarray(states, dtype=np.float64).reshape(-1, 7)
        h.check(h.lib.artp_roadmap_add_milestones(h.h, s.ctypes.data, s.shape[0]))

    def sampleGraph(self, sampler: SE3FromSE2Sampler, max_n_vertices: int = 10000, max_n_edges: int = 50000,
                    recompute_density_after_n_samples: int = 1000, max_draws: int = 1 << 26, first_sample: int = 0,
                    distribution: bool = True) -> int:
        """PRMMotionCostMaintainer::sampleGraph's loop with `sampler`'s Philox stream from first_sample; the distribution is
        re-applied from `sampler`'s parameters (SE3FromSE2Sampler.updateDistribution) unless distribution=False. A draw
        budget replaces max_sample_time. Returns the draws used."""
        h = self._c.handle
        p = capi.ArtpRoadmapParams(int(max_n_vertices), int(max_n_edges), int(recompute_density_after_n_samples), int(max_draws))
        dp = _distribution_params(sampler._sp, h.params) if distribution else None
        used = C.c_uint64(0)
        h.check(h.lib.artp_roadmap_sample_graph(h.h, C.byref(p), None if dp is None else C.byref(dp), sampler.seed,
                                                int(first_sample), C.byref(used)))
        return used.value

    def counts(self):
        h = self._c.handle
        nv, ne = C.c_size_t(0), C.c_size_t(0)
        h.check(h.lib.artp_roadmap_get(h.h, 0, None, None, 0, None, C.byref(nv), C.byref(ne)))
        return nv.value, ne.value

    def vertices(self, first: int = 0):
        """(states [V - first, 7] float64, kinds [V - first] uint8) of the vertices first .. V-1."""
        h = self._c.handle
        nv, _ = self.counts()
        n = max(nv - int(first), 0)
        states, kinds = np.empty((n, 7), np.float64), np.empty(n, np.uint8)
        h.check(h.lib.artp_roadmap_get(h.h, int(first), states.ctypes.data, kinds.ctypes.data, 0, None, None, None))
        return states, kinds

    def edges(self, first: int = 0):
        """[E - first, 2] uint32 (u, v) of the edges first .. E-1."""
        h = self._c.handle
        _, ne = self.counts()
        e = np.empty((max(ne - int(first), 0), 2), np.uint32)
        h.check(h.lib.artp_roadmap_get(h.h, 0, None, None, int(first), e.ctypes.data, None, None))
        return e

    def updateEdges(self) -> None:
        """PRMMotionCostMaintainer::updateEdges (:27-73) over the whole store, on the device."""
        h = self._c.handle
        h.check(h.lib.artp_roadmap_update_edges(h.h))

    def solve(self, start, goal, space, path_capacity: int = 4096):
        """One query (clearQuery + PRMMotionCost::baseSolve) on the device. space: MotionValidator.se3Space(...).
        Returns (status, path states [n, 7] from start to goal, their vertex indices [n], cost, info); the path is empty
        unless status == SOLVED. info: searches, sweeps, edges_checked, edges_removed, start_vertex, goal_vertex."""
        h = self._c.handle
        a = np.ascontiguousarray(start, dtype=np.float64).reshape(7)
        b = np.ascontiguousarray(goal, dtype=np.float64).reshape(7)
        states, idx = np.empty((int(path_capacity), 7), np.float64), np.empty(int(path_capacity), np.uint32)
        n, cost = C.c_size_t(0), C.c_double(0.0)
        info = capi.ArtpRoadmapSolveInfo()
        info.path_vertices = idx.ctypes.data
        h.check(h.lib.artp_roadmap_solve(h.h, a.ctypes.data, b.ctypes.data, C.byref(space), states.ctypes.data, int(path_capacity),
                                         C.byref(n), C.byref(cost), C.byref(info)))
        out = {k: int(getattr(info, k)) for k in ("searches", "sweeps", "edges_checked", "edges_removed", "start_vertex", "goal_vertex")}
        return int(info.status), states[:n.value].copy(), idx[:n.value].copy(), float(cost.value), out

    def edgeCosts(self, first: int = 0):
        """(cost float64 [E - first], flags uint8 [E - first] of EDGE_VALID / EDGE_REMOVED, live edges in the store)."""
        h = self._c.handle
        _, ne = self.counts()
        m = max(ne - int(first), 0)
        cost, flags = np.empty(m, np.float64), np.empty(m, np.uint8)
        live = C.c_size_t(0)
        h.check(h.lib.artp_roadmap_get_edge_costs(h.h, int(first), cost.ctypes.data, flags.ctypes.data, C.byref(live)))
        return cost, flags, live.value


class PathSimplifier:
    """OMPL 1.4.2's PathSimplifier::simplifyMax and Planner::getSolutionPath(true) (planner.cpp:266-298) on the device
    (artp_simplify_path; the rules are oracle/path_simplify_oracle.py's). space: MotionValidator.se3Space(...) -- the
    motion checks' segment counts. objective: "learned" (MotionCostObjective, needs weights and features) or
    "path_length" (getObjective's PathLengthObjective): the final comparison's cost. seed: the Philox "ARTS" stream
    that replaces OMPL's RNG."""

    OBJECTIVES = {"learned": capi.ARTP_OBJ_LEARNED, "path_length": capi.ARTP_OBJ_PATH_LENGTH}

    def __init__(self, checker: StateValidityChecker, space, objective: str = "learned", seed: int = 0,
                 max_query_edge_length: float = 0.5):
        self._c = checker
        self.space = space
        self.objective = objective
        self.seed = int(seed)
        self.max_query_edge_length = float(max_query_edge_length)   # the learned objective's piece length

    def _run(self, path, objective=None):
        h = self._c.handle
        p = np.ascontiguousarray(path, dtype=np.float64).reshape(-1, 7)
        cap = 256 * p.shape[0] + 64      # the longest path the schedule can leave
        out = np.empty((cap, 7), np.float64)
        n = C.c_size_t(0)
        info = capi.ArtpSimplifyInfo()
        h.check(h.lib.artp_simplify_path(h.h, p.ctypes.data, p.shape[0], C.byref(self.space),
                                         self.OBJECTIVES[self.objective] if objective is None else objective,
                                         self.max_query_edge_length, self.seed, out.ctypes.data, cap, C.byref(n), C.byref(info)))
        d = {k: getattr(info, k) for k, _ in capi.ArtpSimplifyInfo._fields_}
        return out[:n.value].copy(), {k: (float(v) if isinstance(v, float) else int(v)) for k, v in d.items()}

    def getSolutionPath(self, path, simplify: bool = True):
        """(states [n, 7], info): the simplified path unless its check fails or the original is strictly cheaper.
        simplify=False returns the path unchanged (and info None), like the reference's flag."""
        if not simplify:
            return np.array(path, dtype=np.float64).reshape(-1, 7), None
        return self._run(path)

    def simplifyMax(self, path):
        """(states [n, 7], info): the simplified path whenever it passes the check (no cost comparison), else the
        original."""
        return self._run(path, capi.ARTP_OBJ_NONE)


class Planner:
    """art_planner::Planner for planner.name prm_motion_cost (planner.cpp:135-298) on the device: setMap is
    artp_planner_set_map, plan is artp_plan (with getSolutionPath's simplification when params.simplify), and every stage
    hands its data to the next in device memory. params: a capi.ArtpPlannerParams (Planner.params() builds one from the
    shipped values). The learned objective needs MotionCostObjective(checker).setWeights first."""

    UNKNOWN, INVALID_START, INVALID_GOAL, NO_MAP, NOT_SOLVED, SOLVED = range(6)   # PlannerStatus (planner_status.h)

    def __init__(self, checker: StateValidityChecker, params):
        self._c = checker
        self.parameters = params
        self._path, self._solved, self._info = None, False, None

    @staticmethod
    def params(seed: int = 0, **kw):
        """An ArtpPlannerParams with the shipped values (params.yaml, params.h) and `kw` overrides; the Basic fields may be
        given as basic=BasicParams-like object."""
        p = capi.ArtpPlannerParams()
        d = dict(start_radius=0.2, goal_radius=0.5, n_iter=1000, max_n_vertices=10000, max_n_edges=50000,
                 recompute_density_after_n_samples=1000, max_query_edge_length=0.5, max_draws=1 << 26, vertex_capacity=20000,
                 edge_capacity=60000, max_roll_pert=3.33 / 180 * np.pi, max_pitch_pert=10.0 / 180 * np.pi,
                 sample_from_distribution=1, use_inverse_vertex_density=1, use_max_prob_unknown_samples=1,
                 max_prob_unknown_samples=0.1, simplify=1, clear_roadmap=0, seed=int(seed), cost_map_from_raw=0)
        basic = kw.pop("basic", None)
        d.update(kw)
        for k, v in d.items():
            setattr(p, k, v)
        b = basic if basic is not None else type("B", (), dict(traversability_thres=0.15, unknown_space_untraversable=1,
                                                                 foothold_margin=0.3, foothold_margin_max_hole_size=0.3,
                                                                 foothold_margin_max_drop=0.3,
                                                                 foothold_margin_max_drop_search_radius=0.16,
                                                                 foothold_margin_min_step=0.3, foothold_size=0.1))
        p.basic = capi.basic_params(b)
        return p

    def setMap(self, elevation, traversability, elevation_inpainted, traversability_inpainted, res: float, cx: float,
               cy: float) -> dict:
        """Planner::setMap + the new-map chain. elevation / traversability: the RAW layers (NaN = unknown; traversability
        may be None); *_inpainted: what inpaintMatrix returned for them (None with a None traversability). Returns the
        call's host_syncs, bytes_h2d and bytes_d2h."""
        f = lambda a: None if a is None else np.asfortranarray(a, dtype=np.float32)
        e, t, ei, ti = f(elevation), f(traversability), f(elevation_inpainted), f(traversability_inpainted)
        h = self._c.handle
        mi = capi.ArtpPlannerMapInfo()
        h.check(h.lib.artp_planner_set_map(h.h, C.byref(self.parameters), *[None if a is None else a.ctypes.data for a in (e, t, ei, ti)],
                                           e.shape[0], e.shape[1], float(res), float(cx), float(cy), C.byref(mi)))
        return {k: int(getattr(mi, k)) for k, _ in capi.ArtpPlannerMapInfo._fields_}

    def setMapRaw(self, elevation, traversability, res: float, cx: float, cy: float) -> dict:
        """setMap from the RAW layers alone (artp_planner_set_map_raw): processors::Basic's two inpaintMatrix calls run
        on the device. traversability may be None. Returns the call's host_syncs, bytes_h2d and bytes_d2h."""
        e = np.asfortranarray(elevation, dtype=np.float32)
        t = None if traversability is None else np.asfortranarray(traversability, dtype=np.float32)
        h = self._c.handle
        mi = capi.ArtpPlannerMapInfo()
        h.check(h.lib.artp_planner_set_map_raw(h.h, C.byref(self.parameters), e.ctypes.data, None if t is None else t.ctypes.data,
                                               e.shape[0], e.shape[1], float(res), float(cx), float(cy), C.byref(mi)))
        return {k: int(getattr(mi, k)) for k, _ in capi.ArtpPlannerMapInfo._fields_}

    def space(self):
        """The artp_se3_space setMap installed (capi.ArtpSe3Space)."""
        sp = capi.ArtpSe3Space()
        self._c.handle.check(self._c.handle.lib.artp_planner_get_space(self._c.handle.h, C.byref(sp)))
        return sp

    def plan(self, start, goal, capacity: int = 1 << 16) -> int:
        """Planner::plan (+ getSolutionPath's simplification when the params say so): returns the PlannerStatus."""
        h = self._c.handle
        a = np.ascontiguousarray(start, dtype=np.float64).reshape(7)
        b = np.ascontiguousarray(goal, dtype=np.float64).reshape(7)
        self._solved, self._path, self._info = False, None, None   # a failing call leaves no solution behind
        out = np.empty((int(capacity), 7), np.float64)
        n = C.c_size_t(0)
        info = capi.ArtpPlanInfo()
        h.check(h.lib.artp_plan(h.h, C.byref(self.parameters), a.ctypes.data, b.ctypes.data, out.ctypes.data, int(capacity),
                                C.byref(n), C.byref(info)))
        self._info = info
        self._solved = info.status == self.SOLVED
        self._path = out[:n.value].copy()
        return int(info.status)

    def getSolutionPath(self):
        """The last plan's path [n, 7] (simplified when the params said so); raises like planner.cpp:268-270 when the
        plan did not solve."""
        if not self._solved:
            raise RuntimeError("Requested failed solution path.")
        return self._path

    def info(self) -> dict:
        """The last plan's artp_plan_info as a dict (nested solve / simplify dicts, 7-vectors as arrays)."""
        def conv(s):
            out = {}
            for k, _ in s._fields_:
                v = getattr(s, k)
                if isinstance(v, C.Structure):
                    v = conv(v)
                elif isinstance(v, C.Array):
                    v = np.array(v[:])
                out[k] = v
            return out
        d = conv(self._info)
        d["solve"].pop("path_vertices", None)
        return d


class StartState:
    """art_planner::StartState (start.h, start.cpp:7-41): the start pose repaired by a disc search around it, one device
    call per sampleGoal. Offsets come from the Philox "ARTB" stream of `seed`; the draw position advances by what the
    reference's loop consumes: k draws when candidate k is returned, n_iter when none is valid, none for a valid centre."""

    def __init__(self, checker: StateValidityChecker, seed: int = 0):
        self._c = checker
        self.seed = int(seed)
        self.draw = 0
        self._state = None
        self.threshold = 0.0
        self.max_num_samples = 0

    def setState(self, state) -> None:
        self._state = np.array(state, dtype=np.float64).reshape(7)

    def setThreshold(self, threshold: float) -> None:
        self.threshold = float(threshold)

    def setMaxNumSamples(self, n: int) -> None:
        self.max_num_samples = int(n)

    def sampleGoal(self, state=None):
        """The repaired state (written into `state` [7] if given) and its candidate index (-1: none valid; the state is
        then the last candidate drawn, like the reference)."""
        out, idx = self._c.findValidNear(self._state.reshape(1, 7), self.threshold, self.max_num_samples, seed=self.seed,
                                         first_draw=self.draw)
        k = int(idx[0])
        self.draw += k if k >= 0 else self.max_num_samples
        if state is not None:
            state[:] = out[0]
            return state, k
        return out[0], k


class GoalStateRegion(StartState):
    """art_planner::GoalStateRegion (goal.h, goal.cpp:11-41): the same search, called by OMPL from inside solve()."""


class MotionValidator:
    """Discrete motion validation over StateValidityChecker (OMPL DiscreteMotionValidator semantics with a fixed
    segment count): valid(s2) and valid(interpolate(s1, s2, j/(n_steps+1))) for j = 1..n_steps."""

    def __init__(self, checker: StateValidityChecker, n_steps: int = 20):
        self._c = checker
        self.n_steps = int(n_steps)

    def checkMotion(self, s1, s2) -> bool:
        a = np.ascontiguousarray(s1, dtype=np.float64).reshape(1, 7)
        b = np.ascontiguousarray(s2, dtype=np.float64).reshape(1, 7)
        return bool(self.checkMotionBatch(a, b)[0])

    def checkMotionBatch(self, s1, s2, out=None):
        h, lib = self._c.handle, self._c.handle.lib
        if _is_torch_cuda(s1):
            import torch
            assert s1.dtype == torch.float64 and s2.dtype == torch.float64 and s1.is_contiguous() and s2.is_contiguous()
            n = s1.shape[0]
            if out is None:
                out = torch.empty(n, dtype=torch.uint8, device=s1.device)
            h.check(lib.artp_check_motions_device(h.h, C.c_void_p(s1.data_ptr()), C.c_void_p(s2.data_ptr()), n,
                                                  self.n_steps, C.c_void_p(out.data_ptr()), _stream_ptr()))
            return out
        a = np.ascontiguousarray(s1, dtype=np.float64)
        b = np.ascontiguousarray(s2, dtype=np.float64)
        n = a.shape[0]
        if out is None:
            out = np.empty(n, dtype=np.uint8)
        h.check(lib.artp_check_motions(h.h, a.ctypes.data, b.ctypes.data, n, self.n_steps, out.ctypes.data))
        return out

    @staticmethod
    def se3Space(synth_map, reach_z: float, fraction: float = 0.01):
        """The SE3 space parameters Planner::setMap installs (planner.cpp:146-156): x, y bounds = map centre +- the FULL
        map length, z bounds = finite elevation range -+ reach.z / 2; OMPL's default longest-valid-segment fraction."""
        lx, ly = synth_map.length
        e = synth_map.elevation[np.isfinite(synth_map.elevation)]
        return capi.ArtpSe3Space((C.c_double * 3)(synth_map.cx - lx, synth_map.cy - ly, float(e.min()) - reach_z / 2),
                                 (C.c_double * 3)(synth_map.cx + lx, synth_map.cy + ly, float(e.max()) + reach_z / 2), float(fraction))

    def validSegmentCount(self, space, s1, s2):
        """SE3StateSpace::validSegmentCount per edge (OMPL 1.4.2 rule, host arithmetic)."""
        a = np.ascontiguousarray(s1, dtype=np.float64); b = np.ascontiguousarray(s2, dtype=np.float64)
        nd = np.empty(a.shape[0], np.int32)
        self._c.handle.check(self._c.handle.lib.artp_valid_segment_count(C.byref(space), a.ctypes.data, b.ctypes.data, a.shape[0],
                                                                         nd.ctypes.data))
        return nd

    def checkMotionSegments(self, s1, s2, nd=None, space=None):
        """DiscreteMotionValidator::checkMotion(s1, s2, lastValid) for a batch with per-edge segment counts (nd, or the OMPL
        rule from `space`): returns (valid uint8 [n], lastValid.second float64 [n])."""
        h, lib = self._c.handle, self._c.handle.lib
        a = np.ascontiguousarray(s1, dtype=np.float64); b = np.ascontiguousarray(s2, dtype=np.float64)
        n = a.shape[0]
        seg = None if nd is None else np.ascontiguousarray(nd, dtype=np.int32)
        valid = np.empty(n, np.uint8); t = np.empty(n, np.float64)
        h.check(lib.artp_check_motions_segments(h.h, a.ctypes.data, b.ctypes.data, n, None if seg is None else seg.ctypes.data,
                                                None if space is None else C.byref(space), valid.ctypes.data, t.ctypes.data))
        return valid, t

    def checkEdgeInteriors(self, s1, s2, n_interp=None, max_lateral: float = 0.5):
        """PRMMotionCost::addValidMilestone's connection loop (prm_motion_cost.cpp:341-372) over a batch of candidate
        edges: per edge the number of leading valid interior states (== n_interp[e] iff the connection is valid).
        Returns (valid_prefix, n_interp). Host arrays, or CUDA float64 tensors (then n_interp must be given as an
        int tensor / array and the prefix sums are built with torch)."""
        h, lib = self._c.handle, self._c.handle.lib
        if _is_torch_cuda(s1):
            import torch
            assert s1.dtype == torch.float64 and s2.dtype == torch.float64 and s1.is_contiguous() and s2.is_contiguous()
            n = s1.shape[0]
            if n_interp is None:
                d = torch.sqrt((s2[:, 0] - s1[:, 0]) ** 2 + (s2[:, 1] - s1[:, 1]) ** 2)
                n_interp = (d / max_lateral).to(torch.int64)
            ni = torch.as_tensor(n_interp, device=s1.device).to(torch.int64)
            off = torch.zeros(n + 1, dtype=torch.int64, device=s1.device)
            off[1:] = torch.cumsum(ni, 0)
            total = int(off[-1].item())
            off32 = off.to(torch.int32).contiguous()      # same bits as uint32 below 2^31
            assert total < 2 ** 31
            flags = torch.empty(max(total, 1), dtype=torch.uint8, device=s1.device)
            out = torch.empty(n, dtype=torch.int32, device=s1.device)
            h.check(lib.artp_check_edge_interiors_device(
                h.h, C.c_void_p(s1.data_ptr()), C.c_void_p(s2.data_ptr()), n, C.c_void_p(off32.data_ptr()), total,
                C.c_void_p(flags.data_ptr()), C.c_void_p(out.data_ptr()), _stream_ptr()))
            return out, ni.to(torch.int32)
        a = np.ascontiguousarray(s1, dtype=np.float64)
        b = np.ascontiguousarray(s2, dtype=np.float64)
        n = a.shape[0]
        out = np.empty(n, dtype=np.int32)
        if n_interp is None:
            d = np.sqrt((b[:, 0] - a[:, 0]) ** 2 + (b[:, 1] - a[:, 1]) ** 2)
            ni = (d / max_lateral).astype(np.uint32).astype(np.int32)
        else:
            ni = np.ascontiguousarray(n_interp, dtype=np.int32)
        h.check(lib.artp_check_edge_interiors(h.h, a.ctypes.data, b.ctypes.data, n,
                                              None if n_interp is None else ni.ctypes.data, float(max_lateral),
                                              out.ctypes.data))
        return out, ni


class PathLengthObjective:
    """art_planner::PathLengthObjective::motionCost (path_length_objective.cpp:26-70), batched."""

    def __init__(self, checker: StateValidityChecker):
        self._c = checker

    def motionCost(self, s1, s2) -> float:
        a = np.ascontiguousarray(s1, dtype=np.float64).reshape(1, 7)
        b = np.ascontiguousarray(s2, dtype=np.float64).reshape(1, 7)
        return float(self.motionCostBatch(a, b)[0])

    def motionCostBatch(self, s1, s2, out=None):
        h, lib = self._c.handle, self._c.handle.lib
        if _is_torch_cuda(s1):
            import torch
            n = s1.shape[0]
            if out is None:
                out = torch.empty(n, dtype=torch.float64, device=s1.device)
            h.check(lib.artp_path_length_cost_device(h.h, C.c_void_p(s1.data_ptr()), C.c_void_p(s2.data_ptr()), n,
                                                     C.c_void_p(out.data_ptr()), _stream_ptr()))
            return out
        a = np.ascontiguousarray(s1, dtype=np.float64)
        b = np.ascontiguousarray(s2, dtype=np.float64)
        n = a.shape[0]
        if out is None:
            out = np.empty(n, dtype=np.float64)
        h.check(lib.artp_path_length_cost(h.h, a.ctypes.data, b.ctypes.data, n, out.ctypes.data))
        return out


class MotionCostObjective:
    """art_planner::MotionCostObjective's batch cost functor (objectives/motion_cost_objective.h:22-66,
    motion_cost_objective.cpp:28-33) backed by the on-device network instead of the ROS cost server
    (art_planner_ros/src/planner_ros.cpp:283-308)."""

    def __init__(self, checker: StateValidityChecker):
        self._c = checker

    def setWeights(self, state_dict) -> None:
        """Parameters keyed like the reference module's state_dict (numpy arrays or torch tensors) of either
        network_light or network: a torch.load of either kind of .pt goes straight in. The state dict picks the network
        (init_conv1 has 24 or 32 output channels); call updateFeatures again after a change of network."""
        from . import costnet
        sd = {k: (v.detach().cpu().numpy() if hasattr(v, "detach") else np.asarray(v)) for k, v in state_dict.items()}
        blob = costnet.pack_blob(sd)
        h = self._c.handle
        assert blob.size == h.lib.artp_cost_weights_size_for(costnet.NETWORKS[costnet.network_of(sd)][1])
        h.check(h.lib.artp_set_cost_weights(h.h, blob.ctypes.data, blob.size))

    def network(self) -> str:
        """"light" (network_light.py) or "full" (network.py): the architecture of the loaded weights."""
        from . import costnet
        h = self._c.handle
        net = C.c_int()
        h.check(h.lib.artp_get_cost_network(h.h, C.byref(net)))
        return next(name for name, (_, v) in costnet.NETWORKS.items() if v == net.value)

    def updateFeatures(self) -> None:
        """CostPredictor.updateFeatures over the checker's current map (predictor.py:28-36)."""
        h = self._c.handle
        h.check(h.lib.artp_update_features(h.h))

    def updateFeaturesRaw(self, layer, res: float, cx: float, cy: float) -> None:
        """CostPredictor.updateFeatures on the map the cost server prepares from the RAW rows x cols elevation layer
        (cost_query_server.py _elvMapProcess, artp_update_features_raw): no installed map needed; geometry res, cx, cy.
        numpy arrays use the host entry point, CUDA tensors (column-major float32, as StateValidityChecker.inpaint) the
        device one on the current stream."""
        h = self._c.handle
        if _is_torch_cuda(layer):
            rows, cols = _column_major_cuda(layer, "updateFeaturesRaw")
            h.check(h.lib.artp_update_features_raw_device(h.h, layer.data_ptr(), rows, cols, float(res), float(cx), float(cy),
                                                          _stream_ptr()))
            return
        a = np.asfortranarray(layer, dtype=np.float32)
        h.check(h.lib.artp_update_features_raw(h.h, a.ctypes.data, a.shape[0], a.shape[1], float(res), float(cx), float(cy)))

    def costMap(self, layer):
        """The cost server's preparation of the RAW rows x cols elevation layer (artp_cost_map_layer): the map whose
        network input the server feeds the trunk, in grid_map layout, column-major float32. A CUDA tensor (column-major,
        as StateValidityChecker.inpaint) gives a CUDA tensor of the same layout, on the current stream."""
        h = self._c.handle
        if _is_torch_cuda(layer):
            import torch
            rows, cols = _column_major_cuda(layer, "costMap")
            out = torch.empty((cols, rows), dtype=torch.float32, device=layer.device).t()
            h.check(h.lib.artp_cost_map_layer_device(h.h, layer.data_ptr(), rows, cols, out.data_ptr(), _stream_ptr()))
            return out
        a = np.asfortranarray(layer, dtype=np.float32)
        out = np.empty(a.shape, np.float32, order="F")
        h.check(h.lib.artp_cost_map_layer(h.h, a.ctypes.data, a.shape[0], a.shape[1], out.ctypes.data))
        return out

    def costQuery(self, edge_matrix, out=None):
        """edge_matrix [n, 6] float32 = [tx, ty, tyaw, sx, sy, syaw] -> [n, 3] float32 (energy, time, risk)."""
        h, lib = self._c.handle, self._c.handle.lib
        if _is_torch_cuda(edge_matrix):
            import torch
            assert edge_matrix.dtype == torch.float32 and edge_matrix.is_contiguous()
            n = edge_matrix.shape[0]
            if out is None:
                out = torch.empty((n, 3), dtype=torch.float32, device=edge_matrix.device)
            h.check(lib.artp_motion_cost_device(h.h, C.c_void_p(edge_matrix.data_ptr()), n, C.c_void_p(out.data_ptr()),
                                                _stream_ptr()))
            return out
        e = np.ascontiguousarray(edge_matrix, dtype=np.float32)
        n = e.shape[0]
        if out is None:
            out = np.empty((n, 3), dtype=np.float32)
        h.check(lib.artp_motion_cost(h.h, e.ctypes.data, n, out.ctypes.data))
        return out

    def edgeMatrixFromStates(self, s_start, s_target):
        """[n, 6] float32 rows [tx, ty, tyaw, sx, sy, syaw] as PRMMotionCostMaintainer::updateEdges fills them."""
        a = np.ascontiguousarray(s_start, dtype=np.float64); b = np.ascontiguousarray(s_target, dtype=np.float64)
        out = np.empty((a.shape[0], 6), np.float32)
        self._c.handle.check(self._c.handle.lib.artp_edge_matrix_from_states(a.ctypes.data, b.ctypes.data, a.shape[0], out.ctypes.data))
        return out

    def updateEdgesBatch(self, s_start, s_target):
        """PRMMotionCostMaintainer::updateEdges / computeCostForVertexEdges for n graph edges in one call: edge matrix ->
        cost query -> isFeasible / getCost. Returns (cost float64 [n] with +inf for infeasible edges, feasible uint8 [n],
        cost3 float32 [n, 3])."""
        h = self._c.handle
        a = np.ascontiguousarray(s_start, dtype=np.float64); b = np.ascontiguousarray(s_target, dtype=np.float64)
        n = a.shape[0]
        cost = np.empty(n, np.float64); feas = np.empty(n, np.uint8); c3 = np.empty((n, 3), np.float32)
        h.check(h.lib.artp_motion_cost_states(h.h, a.ctypes.data, b.ctypes.data, n, cost.ctypes.data, feas.ctypes.data, c3.ctypes.data))
        return cost, feas, c3

    def motionCost(self, s1, s2) -> float:
        """MotionCostObjective::motionCost (motion_cost_objective.cpp:36-95) of one edge: a batch of one."""
        a = np.ascontiguousarray(s1, dtype=np.float64).reshape(1, 7)
        b = np.ascontiguousarray(s2, dtype=np.float64).reshape(1, 7)
        return float(self.motionCostBatch(a, b)[0])

    def motionCostBatch(self, s1, s2, max_query_edge_length: float = 0.5, out=None, rows=None, cost3=None):
        """MotionCostObjective::motionCost for n edges [n, 7] -> float64 [n]: each edge split into
        (unsigned)(lateralDistance / max_query_edge_length) + 1 pieces, every piece queried, +inf if a piece is too
        risky, else the ordered sum of getCost. numpy arrays use the host entry point; CUDA float64 tensors the device
        entry point on the current stream, with the per-edge piece offsets built by torch. rows [>= pieces, 6] float32
        and cost3 [>= pieces, 3] float32 (CUDA only, optional) receive the piece rows and their (energy, time, risk)."""
        h, lib = self._c.handle, self._c.handle.lib
        if _is_torch_cuda(s1):
            import torch
            assert s1.dtype == torch.float64 and s2.dtype == torch.float64 and s1.is_contiguous() and s2.is_contiguous()
            if not max_query_edge_length > 0:
                raise capi.ArtpError(capi.ARTP_E_INVALID, "max_query_edge_length must be > 0")
            n = s1.shape[0]
            if out is None:
                out = torch.empty(n, dtype=torch.float64, device=s1.device)
            if n == 0:
                return out
            d = torch.sqrt((s2[:, 0] - s1[:, 0]) ** 2 + (s2[:, 1] - s1[:, 1]) ** 2)   # lateralDistance, utils.h:52-61
            q = d / max_query_edge_length
            if not bool((q < 2.0 ** 32).all()):
                raise capi.ArtpError(capi.ARTP_E_INVALID, "edge too long or not finite (n_interp must fit 32 bits)")
            off = torch.zeros(n + 1, dtype=torch.int64, device=s1.device)
            off[1:] = torch.cumsum(q.to(torch.int64) + 1, 0)
            total = int(off[-1].item())
            if total >= 2 ** 32:
                raise capi.ArtpError(capi.ARTP_E_INVALID, "too many pieces (>= 2^32)")
            off32 = off.to(torch.int32)      # two's-complement wrap: the uint32 offsets' bits
            if rows is None:
                rows = torch.empty((total, 6), dtype=torch.float32, device=s1.device)
            if cost3 is None:
                cost3 = torch.empty((total, 3), dtype=torch.float32, device=s1.device)
            assert rows.shape[0] >= total and cost3.shape[0] >= total and rows.is_contiguous() and cost3.is_contiguous()
            h.check(lib.artp_motion_cost_split_device(
                h.h, C.c_void_p(s1.data_ptr()), C.c_void_p(s2.data_ptr()), n, C.c_void_p(off32.data_ptr()), total,
                C.c_void_p(rows.data_ptr()), C.c_void_p(cost3.data_ptr()), C.c_void_p(out.data_ptr()), _stream_ptr()))
            return out
        a = np.ascontiguousarray(s1, dtype=np.float64)
        b = np.ascontiguousarray(s2, dtype=np.float64)
        n = a.shape[0]
        if out is None:
            out = np.empty(n, dtype=np.float64)
        h.check(lib.artp_motion_cost_split(h.h, a.ctypes.data, b.ctypes.data, n, float(max_query_edge_length),
                                           out.ctypes.data))
        return out

    def pathCost(self, states, max_query_edge_length: float = 0.5) -> float:
        """PathGeometric::cost(obj) for this objective (OMPL 1.4.2): 0 for fewer than two states, else the left-to-right
        sum of motionCost over consecutive states (initial and terminal cost are the identity 0), one batch call."""
        if len(states) < 2:
            return 0.0
        c = self.motionCostBatch(states[:-1], states[1:], max_query_edge_length)
        total = 0.0
        for v in c.tolist():   # not sum(): Python's float sum is compensated, the reference's is not
            total += v
        return total

    def getCost(self, cost3):
        """(cost, feasible) per edge: w_e*E + w_t*T + w_r*R and R <= risk_threshold (motion_cost_objective.h:54-66)."""
        h = self._c.handle
        c = np.ascontiguousarray(cost3, dtype=np.float32)
        n = c.shape[0]
        cost = np.empty(n, dtype=np.float64)
        feas = np.empty(n, dtype=np.uint8)
        h.check(h.lib.artp_combine_cost(h.h, c.ctypes.data, n, cost.ctypes.data, feas.ctypes.data))
        return cost, feas

    def features(self):
        """[Hf, Wf, C] float32 feature map (test hook); C = 48 for network_light, 64 for network."""
        from . import costnet
        h = self._c.handle
        hf, wf = C.c_int(), C.c_int()
        h.check(h.lib.artp_get_features(h.h, None, 0, C.byref(hf), C.byref(wf)))
        ch = costnet.NETWORKS[self.network()][0][5][2]   # init_flatten's output channels
        out = np.empty((hf.value, wf.value, ch), dtype=np.float32)
        h.check(h.lib.artp_get_features(h.h, out.ctypes.data, out.size, C.byref(hf), C.byref(wf)))
        return out

    def setMode(self, mode: int) -> None:
        h = self._c.handle
        h.check(h.lib.artp_set_cnn_mode(h.h, int(mode)))

    def lastTrunkTimesMs(self):
        ms = (C.c_float * 3)()
        self._c.handle.check(self._c.handle.lib.artp_get_cnn_timing(self._c.handle.h, ms))
        return float(ms[0]), float(ms[1]), float(ms[2])
