"""``Config`` -- sizes that stay fixed for the lifetime of a planner / TDM pair.

Drop-in for the reference's ``mppi_numba.config.Config`` (config.py:16-100): same keyword
arguments, same derived fields, same clamps.  Differences by design: importing this module does NOT
touch a GPU (the reference queries the device at import, config.py:9-12, SURVEY.md 9-B4); the
limits it used to read from the device are the constants every CUDA device since sm_30 reports.
"""

# Limits the reference read from the device (identical on an H100).
max_threads_per_block = 1024
max_square_block_dim = (32, 32)          # (int(1024**0.5),) * 2
max_blocks = 2 ** 31 - 1
rec_max_control_rollouts = max_rec_blocks = 15000
rec_min_control_rollouts = 100

_MODE_FLAGS = ("use_tdm", "use_det_dynamics", "use_nom_dynamics_with_speed_map", "use_costmap")


def _clamp_with_note(name, value, lo, hi):
    if value > hi:
        print("MPPI Config: {} = {} exceeds the recommended maximum; using {}.".format(name, value, hi))
        return hi
    if value < lo:
        print("MPPI Config: {} = {} is below the minimum; using {}.".format(name, value, lo))
        return lo
    return value


class Config:
    """Planner configuration (horizon, batch sizes, map allocation, RNG seed, planner mode)."""

    def __init__(self, T=10, dt=0.1, num_grid_samples=1024, num_control_rollouts=1024,
                 max_speed_padding=5.0, tdm_sample_thread_dim=(16, 16), num_vis_state_rollouts=20,
                 max_map_dim=(250, 250), seed=1, use_tdm=False, use_det_dynamics=False,
                 use_nom_dynamics_with_speed_map=False, use_costmap=False):
        flags = dict(use_tdm=use_tdm, use_det_dynamics=use_det_dynamics,
                     use_nom_dynamics_with_speed_map=use_nom_dynamics_with_speed_map,
                     use_costmap=use_costmap)
        for k in _MODE_FLAGS:
            setattr(self, k, flags[k])
        assert T > 0 and dt > 0 and T > dt
        assert sum(bool(v) for v in flags.values()) == 1, \
            "MPPI Config Error: exactly one of {} must be true.".format(", ".join(_MODE_FLAGS))
        assert not use_costmap, "Interface with costmap2d is not yet implemented."

        self.seed = seed
        self.T, self.dt = T, dt
        self.num_steps = int(T / dt)
        assert self.num_steps > 0
        self.max_threads_per_block = max_threads_per_block

        # M: sampled traction maps (reference: > 1024 switches to its "oversized" kernel)
        if num_grid_samples > max_threads_per_block:
            print("WARNING: num_grid_samples({})>max_threads_per_block({}): the reference switches to its "
                  "oversized kernel here (mppi.py:199-203), whose CVaR is only meaningful for cvar_alpha=1; this "
                  "engine evaluates the mean of the ceil(M*cvar_alpha) largest costs for any M.".format(
                      num_grid_samples, max_threads_per_block))
        self.num_grid_samples = _clamp_with_note("num_grid_samples", num_grid_samples, 1, max_rec_blocks)
        # N: control sequences
        self.num_control_rollouts = _clamp_with_note("num_control_rollouts", num_control_rollouts,
                                                     rec_min_control_rollouts, rec_max_control_rollouts)
        self.max_speed_padding = max_speed_padding

        assert len(tdm_sample_thread_dim) == 2 and min(tdm_sample_thread_dim) > 0
        self.tdm_sample_thread_dim = tuple(tdm_sample_thread_dim)
        if self.tdm_sample_thread_dim[0] * self.tdm_sample_thread_dim[1] >= max_threads_per_block:
            print("MPPI Config: tdm_sample_thread_dim {} has >= {} threads; using {}.".format(
                tuple(tdm_sample_thread_dim), max_threads_per_block, max_square_block_dim))
            self.tdm_sample_thread_dim = max_square_block_dim

        v = min(num_vis_state_rollouts, self.num_control_rollouts, self.num_grid_samples)
        self.num_vis_state_rollouts = max(1, v)
        self.max_map_dim = max_map_dim

    @property
    def mode(self):
        """0 = use_tdm, 1 = use_det_dynamics, 2 = use_nom_dynamics_with_speed_map (b200mppi.h)."""
        return 1 if self.use_det_dynamics else 2 if self.use_nom_dynamics_with_speed_map else 0

    @property
    def det_dyn(self):
        return self.use_det_dynamics or self.use_nom_dynamics_with_speed_map or self.use_costmap
