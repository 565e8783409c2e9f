"""Traction-distribution maps for the H100 MPPI engine.

``TDM_Numba`` keeps the public surface of the reference class of the same name
(mppi_numba/terrain.py:69-628): the two setters, ``sample_grids``, the padded-limit attributes the
planner and the visualiser read.  The map is stored on the device by libb200mppi.so
(b200mppi_tdm_* in include/b200mppi.h); host-side preparation (CVaR / mean collapse for the
deterministic modes, zero-traction padding, cropping to ``max_map_dim``) is numpy, as in the
reference, but vectorised per terrain class / per grid instead of per cell.

``Terrain`` and ``TractionGrid`` are the small simulation-side helpers (terrain.py:24-66,750-785)
that closed-loop drivers use next to the planner; they never touch the GPU.

``draw_traction_grids(lin_tdm, ang_tdm, count)`` draws ground-truth realisations of a TDM pair on the GPU, as the
reference notebook's ``sample_traction_grid`` helper does, and keeps them there: each ``DeviceTractionGrid`` can be
given to the batches' trial calls wherever a ``TractionGrid`` is taken, and the plant reads it in place.
"""
import ctypes as C
import math
import time

import numpy as np

from . import _lib
from ._lib import DeviceArray, check, lib, ptr


def _host_mirror(owner, host_array):
    """Device array whose content is an immutable upload of ``host_array``."""
    keep = np.ascontiguousarray(host_array)

    def read(out):
        out[...] = keep
    return DeviceArray(owner, keep.shape, keep.dtype, read)


class TDM_Numba(object):
    """Traction Distribution Map: per-cell PMF over traction bins, int8 percent, shape
    (num_bins, rows, cols), padded with a ring of zero-traction cells so that rollouts never need a
    bounds check (reference README.md:164-165).

    Workflow (unchanged): construct with a ``Config`` -> ``reset()`` -> one of the two setters ->
    hand the object to ``MPPI_Numba.setup`` -> repeat from ``reset()`` when the map changes."""

    def __init__(self, cfg, device=0, rank=0, world_size=1):
        """``rank`` / ``world_size``: with ``use_tdm`` and more than one rank the M sampled maps are sharded
        (this object holds maps [rank*M/ws, (rank+1)*M/ws), bit-identical to the same maps of a 1-rank run)."""
        self.cfg = cfg
        self.rank, self.world_size = int(rank), int(world_size)
        for name in ("T", "dt", "num_steps", "num_grid_samples", "num_control_rollouts",
                     "max_speed_padding", "tdm_sample_thread_dim", "num_vis_state_rollouts",
                     "max_map_dim", "seed", "use_tdm", "use_det_dynamics",
                     "use_nom_dynamics_with_speed_map", "use_costmap"):
            setattr(self, name, getattr(cfg, name))
        self.det_dyn = bool(self.use_det_dynamics or self.use_nom_dynamics_with_speed_map or self.use_costmap)
        self.thread_dim = tuple(self.tdm_sample_thread_dim)
        self.block_dim = (1, self.num_grid_samples)
        self.total_threads = self.num_grid_samples * self.thread_dim[0] * self.thread_dim[1]
        self.device = int(device)

        self._handle = None
        self.sample_grid_batch_d = None
        self.risk_traction_map_d = None
        self.obstacle_map_d = None
        self.unknown_map_d = None
        self.rng_states_d = None
        self.device_var_initialized = False
        self.reset()

    # ------------------------------------------------------------------ lifetime
    def __del__(self):
        h, self._handle = getattr(self, "_handle", None), None
        if h:
            try:
                lib.b200mppi_tdm_destroy(h)
            except Exception:
                pass

    def reset(self):
        """Forget the task-specific map (host side).  Like the reference (SURVEY.md 9-Q3) the device
        sample buffer and the RNG streams survive a reset."""
        self.semantic_grid = None
        self.semantic_grid_initialized = False
        self.id2name = self.name2terrain = self.id2terrain_fn = self.terrain2pmf = None
        self.pmf_grid = None
        self.bin_values = self.bin_values_bounds = None
        self.pmf_grid_d = self.bin_values_d = self.bin_values_bounds_d = None
        self.num_pmf_bins = None
        self.xlimits = self.ylimits = None
        self.padded_xlimits = self.padded_ylimits = None
        self.pad_cells = None
        self.res = None
        self.pmf_grid_initialized = False
        self.risk_traction_map_d = None
        self.obstacle_map = self.obstacle_map_d = None
        self.unknown_map = self.unknown_map_d = None
        self.cell_dimensions = None
        self.figsize = None
        self.init_device_vars_before_sampling()

    def init_device_vars_before_sampling(self):
        if self.device_var_initialized:
            return
        t0 = time.time()
        rows, cols = self.max_map_dim
        pod = _lib.ConfigPOD(num_steps=self.num_steps, num_control_rollouts=self.num_control_rollouts,
                             num_grid_samples=self.num_grid_samples, max_map_rows=rows, max_map_cols=cols,
                             tdm_thread_x=self.thread_dim[0], tdm_thread_y=self.thread_dim[1],
                             num_vis_state_rollouts=self.num_vis_state_rollouts, mode=self.cfg.mode,
                             device=self.device, rank=self.rank, world_size=self.world_size,
                             seed=int(self.seed) & (2 ** 64 - 1))
        h = C.c_void_p()
        check(lib.b200mppi_tdm_create(C.byref(pod), C.byref(h)))
        self._handle = h
        maps = 1 if self.det_dyn else self.num_grid_samples // self.world_size
        base, pitch = C.c_void_p(), C.c_int32()
        check(lib.b200mppi_tdm_sample_grid_view(h, C.byref(base), C.byref(pitch)))
        self.sample_grid_batch_d = DeviceArray(
            self, (maps, rows, cols), np.int8,
            lambda out: check(lib.b200mppi_tdm_get_sample_grids(h, ptr(out), out.nbytes)),
            lambda src: check(lib.b200mppi_tdm_set_sample_grids(h, ptr(src), src.nbytes)),
            dev_ptr=lambda: base.value, strides=(rows * pitch.value, pitch.value, 1))
        ngen = C.c_int64()
        check(lib.b200mppi_tdm_num_generators(h, C.byref(ngen)))
        self.rng_states_d = DeviceArray(
            self, (ngen.value, 2), np.uint64,
            lambda out: check(lib.b200mppi_tdm_get_rng_states(h, ptr(out), out.nbytes)),
            lambda src: check(lib.b200mppi_tdm_set_rng_states(h, ptr(src), src.nbytes)))
        self.device_var_initialized = True
        print("TDM has initialized GPU memory after {} s".format(time.time() - t0))

    # ------------------------------------------------------------------ padding (terrain.py:511-583)
    def get_padding_info(self, grid_shape, max_speed_padding, dt, res):
        rows, cols = grid_shape[-2], grid_shape[-1]
        pad_cells = int(np.ceil(max_speed_padding * dt / res))
        room_r = self.max_map_dim[0] - 2 * pad_cells
        room_c = self.max_map_dim[1] - 2 * pad_cells
        if room_r < 1 or room_c < 1:
            print("TDM padding leaves no room for the map: {} x {} usable cells of allocation {}".format(
                room_r, room_c, [1 if self.det_dyn else self.num_grid_samples] + list(self.max_map_dim)))
            assert False
        keep_r, keep_c = min(room_r, rows), min(room_c, cols)
        if keep_r < rows or keep_c < cols:
            print("WARNING: PMF cropped from ({}, {}) to ({}, {}) to fit the allocated map.".format(
                rows, cols, keep_r, keep_c))
        return keep_r, keep_c, pad_cells

    def _padded_limits(self, xlimits, ylimits, keep_r, keep_c, pad, res):
        return (np.array([xlimits[0] - pad * res, xlimits[0] + (keep_c + pad) * res]),
                np.array([ylimits[0] - pad * res, ylimits[0] + (keep_r + pad) * res]))

    def set_padding(self, pmf_grid, max_speed_padding, dt, res, xlimits, ylimits):
        """Crop from the origin corner, surround with ``pad_cells`` cells whose mass sits on bin 0."""
        keep_r, keep_c, pad = self.get_padding_info(pmf_grid.shape, max_speed_padding, dt, res)
        self.pad_cells = pad
        out = np.zeros((pmf_grid.shape[0], keep_r + 2 * pad, keep_c + 2 * pad), dtype=np.int8)
        out[0] = 100
        out[:, pad:pad + keep_r, pad:pad + keep_c] = pmf_grid[:, :keep_r, :keep_c]
        pxl, pyl = self._padded_limits(xlimits, ylimits, keep_r, keep_c, pad, res)
        return out, pxl, pyl

    def set_padding_risk_traction(self, grid, max_speed_padding, dt, res, xlimits, ylimits):
        keep_r, keep_c, pad = self.get_padding_info(grid.shape, max_speed_padding, dt, res)
        self.pad_cells = pad
        out = np.zeros((1, keep_r + 2 * pad, keep_c + 2 * pad), dtype=np.int8)
        out[:, pad:pad + keep_r, pad:pad + keep_c] = grid[:, :keep_r, :keep_c]
        pxl, pyl = self._padded_limits(xlimits, ylimits, keep_r, keep_c, pad, res)
        return out, pxl, pyl

    def set_padding_2d(self, map, max_speed_padding, dt, res, pad_val=0):
        keep_r, keep_c, pad = self.get_padding_info(map.shape, max_speed_padding, dt, res)
        self.pad_cells = pad
        out = np.full((keep_r + 2 * pad, keep_c + 2 * pad), pad_val, dtype=np.int8)
        out[pad:pad + keep_r, pad:pad + keep_c] = map[:keep_r, :keep_c]
        return out

    def get_padded_grid_xy_dim(self):
        if not self.pmf_grid_initialized:
            print("Padded grid has not been initialized yet.")
            return None
        return self.pmf_grid_d.shape[1:]

    def prepare_obstacle_and_unknown_map(self, obstacle_map, unknown_map, num_rows, num_cols, res):
        def as_mask(m, what):
            if m is None:
                return np.zeros((num_rows, num_cols), dtype=np.int8)
            assert m.shape == (num_rows, num_cols), what + " does not have the same XY dim as pmf grid."
            return np.asarray(m).astype(np.int8).reshape(num_rows, num_cols)
        self.obstacle_map = as_mask(obstacle_map, "obstacle_map")
        self.unknown_map = as_mask(unknown_map, "unknown_map")
        obs_p = np.ascontiguousarray(self.set_padding_2d(self.obstacle_map, self.max_speed_padding, self.dt, res))
        unk_p = np.ascontiguousarray(self.set_padding_2d(self.unknown_map, self.max_speed_padding, self.dt, res))
        check(lib.b200mppi_tdm_set_masks(self._handle, ptr(obs_p), ptr(unk_p), obs_p.shape[0], obs_p.shape[1]))
        self.obstacle_map_d = _host_mirror(self, obs_p)
        self.unknown_map_d = _host_mirror(self, unk_p)

    def print_bin_values_bounds(self, obj_name):
        if self.bin_values_bounds_d is None:
            print("{}: Bin value is None".format(obj_name))
        else:
            print("{}: bin values bounds are ".format(obj_name), self.bin_values_bounds_d.copy_to_host())

    # ------------------------------------------------------------------ upload
    def _upload(self, res, xlimits, ylimits, obstacle_map, unknown_map, risk_map=None):
        """Pad + H2D of self.pmf_grid (and masks / risk map); common tail of both setters."""
        num_rows, num_cols = self.pmf_grid.shape[1:]
        if risk_map is not None:
            risk_p, _, _ = self.set_padding_risk_traction(risk_map, self.max_speed_padding, self.dt, res,
                                                          xlimits, ylimits)
        padded, self.padded_xlimits, self.padded_ylimits = self.set_padding(
            self.pmf_grid, self.max_speed_padding, self.dt, res, xlimits, ylimits)
        padded = np.ascontiguousarray(padded)
        bv = np.ascontiguousarray(self.bin_values, dtype=np.float32)
        bb = np.ascontiguousarray(self.bin_values_bounds, dtype=np.float32)
        pxl = np.ascontiguousarray(self.padded_xlimits, dtype=np.float32)
        pyl = np.ascontiguousarray(self.padded_ylimits, dtype=np.float32)
        check(lib.b200mppi_tdm_set_pmf(self._handle, ptr(padded), padded.shape[0], padded.shape[1],
                                       padded.shape[2], ptr(bv), ptr(bb), np.float32(res), ptr(pxl), ptr(pyl)))
        self.pmf_grid_d = _host_mirror(self, padded)
        self.bin_values_d = _host_mirror(self, bv)
        self.bin_values_bounds_d = _host_mirror(self, bb)
        if risk_map is not None:
            r2 = np.ascontiguousarray(risk_p[0])
            check(lib.b200mppi_tdm_set_risk_map(self._handle, ptr(r2), r2.shape[0], r2.shape[1]))
            self.risk_traction_map_d = _host_mirror(self, risk_p)
        self.prepare_obstacle_and_unknown_map(obstacle_map, unknown_map, num_rows, num_cols, res)

    # ------------------------------------------------------------------ setter 1: PMF grid
    def set_TDM_from_PMF_grid(self, pmf_grid, tdm_dict, obstacle_map=None, unknown_map=None):
        """``pmf_grid``: int (num_bins, rows, cols), each column summing to 100.  ``tdm_dict`` keys:
        res, xlimits, ylimits, bin_values, bin_values_bounds, det_dynamics_cvar_alpha."""
        _lib.refuse_in_loop(self, "TDM_Numba.set_TDM_from_PMF_grid")
        alpha = tdm_dict["det_dynamics_cvar_alpha"]
        if not (0 < alpha <= 1.0):
            print("WARNING: TDM cannot be setup since alpha is not in (0,1]")
        assert alpha > 0
        assert alpha <= 1.0
        assert len(pmf_grid.shape) == 3, "PMF grid must have 3 dimensions"
        self.num_pmf_bins, num_rows, num_cols = pmf_grid.shape
        self.res = res = tdm_dict["res"]
        self.cell_dimensions = (res, res)
        self.xlimits, self.ylimits = tdm_dict["xlimits"], tdm_dict["ylimits"]
        self.bin_values = np.asarray(tdm_dict["bin_values"]).astype(np.float32)
        self.bin_values_bounds = np.asarray(tdm_dict["bin_values_bounds"]).astype(np.float32)
        assert self.bin_values[0] == 0, "Assume minimum bin value is 0 for now"
        assert self.bin_values_bounds[0] == 0, "Assume minimum traction is 0 for now"

        if self.use_det_dynamics or self.use_nom_dynamics_with_speed_map:
            # one-map modes: the CVaR / mean collapse (terrain.py:408-495), the crop and the zero-traction
            # padding run on the GPU (b200mppi_tdm_set_pmf_collapsed); the host keeps mirrors of the results
            self._set_collapsed_on_device(np.asarray(pmf_grid), alpha, res, obstacle_map, unknown_map)
        else:
            self.pmf_grid = np.asarray(pmf_grid).astype(np.int8)
            off = np.argwhere(np.sum(self.pmf_grid, axis=0) != 100)
            if len(off):
                print("WARNING: some PMF columns do not sum to 100: {}".format(off))
            self._upload(res, self.xlimits, self.ylimits, obstacle_map, unknown_map, None)
        self.pmf_grid_initialized = True

    def _set_collapsed_on_device(self, pmf_grid, alpha, res, obstacle_map, unknown_map):
        B, num_rows, num_cols = pmf_grid.shape
        keep_r, keep_c, pad = self.get_padding_info(pmf_grid.shape, self.max_speed_padding, self.dt, res)
        self.pad_cells = pad
        self.padded_xlimits, self.padded_ylimits = self._padded_limits(self.xlimits, self.ylimits, keep_r, keep_c, pad, res)
        raw = np.ascontiguousarray(pmf_grid, dtype=np.int8)
        bv = np.ascontiguousarray(self.bin_values, dtype=np.float32)
        bb = np.ascontiguousarray(self.bin_values_bounds, dtype=np.float32)
        pxl = np.ascontiguousarray(self.padded_xlimits, dtype=np.float32)
        pyl = np.ascontiguousarray(self.padded_ylimits, dtype=np.float32)
        Hp, Wp = keep_r + 2 * pad, keep_c + 2 * pad
        padded = np.empty((B, Hp, Wp), dtype=np.int8)
        risk_p = np.empty((1, Hp, Wp), dtype=np.int8) if self.use_nom_dynamics_with_speed_map else None
        bad = C.c_int32(0)
        check(lib.b200mppi_tdm_set_pmf_collapsed(
            self._handle, ptr(raw), B, num_rows, num_cols, keep_r, keep_c, pad, ptr(bv), ptr(bb), np.float32(res),
            ptr(pxl), ptr(pyl), float(alpha), ptr(padded), ptr(risk_p) if risk_p is not None else None, C.byref(bad)))
        if bad.value:
            print("WARNING: the provided PMF has {} columns that don't sum up to 100".format(bad.value))
        self.pmf_grid = padded[:, pad:pad + keep_r, pad:pad + keep_c].copy()
        self.pmf_grid_d = _host_mirror(self, padded)
        self.bin_values_d = _host_mirror(self, bv)
        self.bin_values_bounds_d = _host_mirror(self, bb)
        if risk_p is not None:
            self.risk_traction_map_d = _host_mirror(self, risk_p)
        self.prepare_obstacle_and_unknown_map(obstacle_map, unknown_map, num_rows, num_cols, res)

    # ------------------------------------------------------------------ setter 2: semantic grid
    def set_TDM_from_semantic_grid(self, sg, res, num_pmf_bins, bin_values, bin_values_bounds,
                                   xlimits, ylimits, id2name, name2terrain, terrain2pmf,
                                   det_dynamics_cvar_alpha=None, obstacle_map=None, unknown_map=None):
        """Simulation-benchmark entry: ``sg`` holds semantic ids, ``terrain2pmf[terrain]`` is
        ``(values, pmf)`` with pmf summing to 1.  One PMF column per terrain class is computed and
        broadcast over the cells of that class (the reference loops over cells, terrain.py:226-324)."""
        _lib.refuse_in_loop(self, "TDM_Numba.set_TDM_from_semantic_grid")
        if det_dynamics_cvar_alpha is None:
            assert self.use_tdm or self.use_costmap
        else:
            assert 0 < det_dynamics_cvar_alpha <= 1.0
        self.semantic_grid = sg.copy()
        self.id2name, self.name2terrain, self.terrain2pmf = id2name, name2terrain, terrain2pmf
        self.id2terrain_fn = lambda semantic_id: self.name2terrain[self.id2name[semantic_id]]
        self.semantic_grid_initialized = True
        self.cell_dimensions = (res, res)
        self.xlimits, self.ylimits = xlimits, ylimits
        num_rows, num_cols = sg.shape
        self.num_pmf_bins = num_pmf_bins
        self.bin_values = np.asarray(bin_values).astype(np.float32)
        self.bin_values_bounds = np.asarray(bin_values_bounds).astype(np.float32)
        self.res = res
        assert bin_values[0] == 0, "Assume minimum bin value is 0 for now"
        assert bin_values_bounds[0] == 0, "Assume minimum traction is 0 for now"

        alpha = det_dynamics_cvar_alpha
        self.pmf_grid = np.zeros((num_pmf_bins, num_rows, num_cols), dtype=np.int8)
        span = self.bin_values_bounds[1] - self.bin_values_bounds[0]
        risk_map = np.zeros((1, num_rows, num_cols), dtype=np.int8) if self.use_nom_dynamics_with_speed_map else None
        for sid in np.unique(self.semantic_grid):
            where = self.semantic_grid == sid
            values, pmf = self.terrain2pmf[self.id2terrain_fn(sid)]
            column = np.zeros(num_pmf_bins, dtype=np.int8)
            if self.use_det_dynamics or self.use_nom_dynamics_with_speed_map:
                tail_mass, expected = 0.0, 0.0
                for val, m in zip(values, pmf):          # same accumulation order as the reference
                    tail_mass += m
                    expected += m * val
                    if alpha != 1.0 and tail_mass >= alpha:
                        break
                if alpha != 1.0 and tail_mass > 0:
                    expected /= tail_mass
                if self.use_det_dynamics:
                    for b, vval in enumerate(values):
                        if expected <= vval:
                            column[b] = 100
                            break
                    assert column.sum() == 100
                else:
                    column[-1] = 100
                    risk_map[0][where] = np.int8(100 * (expected - self.bin_values_bounds[0]) / span)
            elif self.use_tdm:
                column[:] = np.int8(np.asarray(pmf) * 100)
                column[-1] = np.int8(100) - np.sum(column[:-1])
                assert column.sum() == 100
            else:
                assert False, "TDM cannot be set up"
            self.pmf_grid[:, where] = column[:, None]
        self._upload(res, xlimits, ylimits, obstacle_map, unknown_map, risk_map)
        raw_bv, raw_bb = np.asarray(bin_values), np.asarray(bin_values_bounds)
        if raw_bv.dtype == np.float64 or raw_bb.dtype == np.float64:
            # the reference uploads bin_values / bounds uncast here (terrain.py:331-332): Numba then
            # evaluates int8(100.*(v-lo)/range) in float64 end to end (0.21 -> 21, not 20)
            q = np.trunc(100.0 * (raw_bv.astype(np.float64) - np.float64(raw_bb[0])) /
                         (np.float64(raw_bb[1]) - np.float64(raw_bb[0]))).astype(np.int64).astype(np.int8)
            q = np.ascontiguousarray(q)
            check(lib.b200mppi_tdm_set_bin_quantisation(self._handle, ptr(q), len(q)))
        Hp, Wp = self.pmf_grid_d.shape[1:]
        self.semantic_grid = self.semantic_grid[:Hp - 2 * self.pad_cells, :Wp - 2 * self.pad_cells].copy()
        self.pmf_grid_initialized = True

    # ------------------------------------------------------------------ sampling
    def sample_grids(self, alpha_dyn=1.0):
        """Sample M (or 1) traction maps from the PMF on the GPU; returns the persistent device array
        (M|1, Rmax, Cmax) int8.  Bit-exact with the reference's generator layout (terrain.py:633-694)."""
        _lib.refuse_in_loop(self, "TDM_Numba.sample_grids")
        check(lib.b200mppi_tdm_sample_grids(self._handle, float(alpha_dyn)))
        return self.sample_grid_batch_d

    def sample_grids_true_dist(self):
        """One traction sample per semantic class from the TRUE densities (not the PMF) ->
        ``TractionGrid`` for the simulated robot (terrain.py:586-608)."""
        lins = np.zeros_like(self.semantic_grid, dtype=float)
        angs = np.zeros_like(self.semantic_grid, dtype=float)
        ids, first, counts = np.unique(np.asarray(self.semantic_grid).ravel(), return_index=True, return_counts=True)
        # classes are visited in order of first appearance (row-major), like the reference's dict walk: with a
        # shared global RNG behind the densities this keeps the draws of every class identical to the reference's
        drawn = {}
        for k in np.argsort(first):
            drawn[ids[k]] = self.id2terrain_fn(ids[k]).sample_traction(int(counts[k]))
        for sid, (lin_s, ang_s) in drawn.items():
            mask = self.semantic_grid == sid
            lins[mask] = lin_s
            angs[mask] = ang_s
        return TractionGrid(lins, angs)

    def int8_grid_to_float32(self, int8grid):
        frac = np.asarray(int8grid.copy()).astype(np.float32) / 100.
        return frac * (self.bin_values_bounds[1] - self.bin_values_bounds[0]) + self.bin_values_bounds[0]


class Terrain(object):
    """Ground-truth traction statistics of one semantic class: the reference's simulation helper
    (terrain.py:24-66), same constructor and attributes.  ``lin_density`` / ``ang_density`` are duck-typed:
    they must offer ``sample(n)``; ``mean(samples)``, ``var(samples)`` and ``cvar(alpha, samples=, front=)``
    (-> (tail mean, threshold), the reference's density.py:25-56) are used when present, numpy otherwise."""

    def __init__(self, name, rgb, lin_density, ang_density, cvar_alpha=0.1, cvar_front=True, num_saved_samples=1e4):
        self.name = name
        self.rgb = rgb
        self.lin_density, self.ang_density = lin_density, ang_density
        self.num_saved_samples = num_saved_samples
        self.lin_saved_samples = np.asarray(lin_density.sample(int(num_saved_samples)))
        self.ang_saved_samples = np.asarray(ang_density.sample(int(num_saved_samples)))
        self.cvar_alpha, self.cvar_front = cvar_alpha, cvar_front
        for axis in ("lin", "ang"):
            dens, smp = getattr(self, axis + "_density"), getattr(self, axis + "_saved_samples")
            mean = dens.mean(smp) if hasattr(dens, "mean") else np.mean(smp)
            var = dens.var(smp) if hasattr(dens, "var") else np.var(smp)
            setattr(self, axis + "_mean", mean)
            setattr(self, axis + "_var", var)
            setattr(self, axis + "_std", np.sqrt(var))
        self.update_cvar_alpha(cvar_alpha)

    @staticmethod
    def _tail(dens, samples, alpha, front):
        """(mean of the alpha-tail, its percentile threshold): the lower tail if ``front``, else the upper one;
        samples equal to the threshold are excluded (density.py:41-56)."""
        if hasattr(dens, "cvar"):
            return dens.cvar(alpha, samples=samples, front=front)
        thres = np.percentile(samples, alpha * 100.0 if front else (1.0 - alpha) * 100.0)
        tail = samples[samples < thres] if front else samples[samples > thres]
        assert tail.size > 0
        return np.mean(tail), thres

    def update_cvar_alpha(self, alpha):
        assert alpha > 0 and alpha <= 1.0
        self.cvar_alpha = alpha
        self.lin_cvar, self.lin_cvar_thres = self._tail(self.lin_density, self.lin_saved_samples, alpha, self.cvar_front)
        self.ang_cvar, self.ang_cvar_thres = self._tail(self.ang_density, self.ang_saved_samples, alpha, self.cvar_front)

    def sample_traction(self, num_samples):
        return self.lin_density.sample(num_samples), self.ang_density.sample(num_samples)

    def __repr__(self):
        return ("Terrain {} has the following properties for linear and angular tractions.\n"
                "mean=({:.2f}, {:.2f}), std=({:.2f}, {:.2f}), cvar({:.2f})=({:.2f}, {:.2f}) "
                "(computed from {} saved samples)").format(
                    self.name, self.lin_mean, self.ang_mean, self.lin_std, self.ang_std, self.cvar_alpha,
                    self.lin_cvar, self.ang_cvar, self.num_saved_samples)


class TractionGrid(object):
    """Deterministic traction grid used by the simulated robot in closed-loop drivers
    (terrain.py:750-785): ``get(x, y)`` -> (linear, angular) traction, 0 outside the map."""

    def __init__(self, lin_traction, ang_traction, res=1.0, use_int8=False, xlimits=None, ylimits=None):
        if use_int8:
            lin_traction = (100 * lin_traction).astype(np.int8)
            ang_traction = (100 * ang_traction).astype(np.int8)
        self.lin_traction, self.ang_traction = lin_traction, ang_traction
        self.res = res
        self.height, self.width = self.lin_traction.shape
        self.xlimits = (0, self.res * self.width) if xlimits is None else xlimits
        self.ylimits = (0, self.res * self.height) if ylimits is None else ylimits

    def get(self, x, y):
        xi = int((x - self.xlimits[0]) // self.res)
        yi = int((y - self.ylimits[0]) // self.res)
        if 0 <= xi < self.width and 0 <= yi < self.height:
            return self.lin_traction[yi, xi], self.ang_traction[yi, xi]
        return 0, 0

    def get_grids(self):
        return self.lin_traction, self.ang_traction


class DeviceTractionGrid(object):
    """One ground-truth realisation in GPU memory, taken by the batches' trial calls wherever a ``TractionGrid`` is:
    the plant step reads its planes in place.  ``res``, ``xlimits``, ``ylimits``, ``height`` and ``width`` as on the
    ``TractionGrid`` the notebook's helper builds; ``get_grids()`` copies both planes to the host.  Keeps its set alive."""

    def __init__(self, owner, index):
        self._owner = owner
        self.index = index
        lin, ang = C.c_void_p(), C.c_void_p()
        check(lib.b200mppi_realisations_planes(owner._handle, index, C.byref(lin), C.byref(ang)))
        self._lin_ptr, self._ang_ptr = lin.value, ang.value
        self.res, self.xlimits, self.ylimits = owner.res, owner.xlimits, owner.ylimits
        self.height, self.width = owner.height, owner.width

    def get_grids(self):
        """(lin, ang): float64 (height, width) host copies of the realisation."""
        lin = np.empty((self.height, self.width), dtype=np.float64)
        ang = np.empty_like(lin)
        check(lib.b200mppi_realisations_copy_out(self._owner._handle, self.index, ptr(lin), ptr(ang)))
        return lin, ang


class DeviceTractionGrids(object):
    """A sequence of ``count`` DeviceTractionGrid drawn by ``draw_traction_grids``; the device memory is freed when
    neither this object nor any of its grids is referenced."""

    def __init__(self, handle, lin_tdm):
        self._handle = handle
        count, height, width, device = C.c_int32(), C.c_int32(), C.c_int32(), C.c_int32()
        check(lib.b200mppi_realisations_info(handle, C.byref(count), C.byref(height), C.byref(width), None, None, None,
                                             C.byref(device)))
        self.height, self.width, self.device = int(height.value), int(width.value), int(device.value)
        # the geometry of the helper's TractionGrid: the TDM's own res and padded limits (float64 on the host)
        self.res = lin_tdm.res
        self.xlimits = np.array(lin_tdm.padded_xlimits, dtype=np.float64)
        self.ylimits = np.array(lin_tdm.padded_ylimits, dtype=np.float64)
        self._grids = [DeviceTractionGrid(self, i) for i in range(int(count.value))]

    def __del__(self):
        h, self._handle = getattr(self, "_handle", None), None
        if h:
            try:
                lib.b200mppi_realisations_destroy(h)
            except Exception:
                pass

    def __len__(self):
        return len(self._grids)

    def __getitem__(self, i):
        return self._grids[i]

    def __iter__(self):
        return iter(self._grids)


def draw_traction_grids(lin_tdm, ang_tdm, count):
    """``count`` ground-truth realisations of the TDM pair, drawn and kept on the GPU: realisation i equals
    ``TractionGrid(lin.astype(np.float64), ang.astype(np.float64), lin_tdm.res, xlimits=lin_tdm.padded_xlimits,
    ylimits=lin_tdm.padded_ylimits)`` for the (lin, ang) of the i-th call of the reference notebook's
    ``sample_traction_grid(lin_tdm, ang_tdm)`` (``sample_grids()`` of each TDM, map 0 as ``q * (hi - lo) / 100.0 + lo``
    in float32), and both TDMs end as after those calls.  ``lin_tdm`` may be ``ang_tdm``.  Returns a
    DeviceTractionGrids.  Raises ValueError for count < 1, a TDM whose PMF is not set and TDMs on different devices."""
    count = int(count)
    if count < 1:
        raise ValueError("draw_traction_grids: count %d < 1" % count)
    for name, t in (("lin_tdm", lin_tdm), ("ang_tdm", ang_tdm)):
        if not t.pmf_grid_initialized:
            raise ValueError("draw_traction_grids: %s has no PMF grid set" % name)
    if lin_tdm.device != ang_tdm.device:
        raise ValueError("draw_traction_grids: lin_tdm is on device %d, ang_tdm on device %d"
                         % (lin_tdm.device, ang_tdm.device))
    h = C.c_void_p()
    check(lib.b200mppi_tdm_draw_realisations(lin_tdm._handle, ang_tdm._handle, count, C.byref(h)))
    return DeviceTractionGrids(h, lin_tdm)
