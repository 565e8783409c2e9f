"""Host restatement of the benchmark's closed-loop episode (TEST INFRASTRUCTURE): the loop MPPI_Batch.run_trials runs
on the device, written out step by step in numpy -- solve, plant step on the ground-truth TractionGrid in float64,
shift_and_update, stop once within goal_tolerance -- plus the trial-log conventions.  Used by the GPU tests and
bench_trials.py as the reference the device episode must reproduce."""
import numpy as np


def plant_step(grid, x, u, dt):
    """(x_next, (lt, at)) for one step from pose x (float64 (3,)) with control u (float32 (2,))."""
    lt, at = grid.get(x[0], x[1])
    xn = np.empty(3)
    xn[0] = x[0] + dt * lt * np.cos(x[2]) * u[0]
    xn[1] = x[1] + dt * lt * np.sin(x[2]) * u[0]
    xn[2] = x[2] + dt * at * u[1]
    return xn


def within(p, x):
    return (p.lin_tdm.padded_xlimits[0] <= x[0] <= p.lin_tdm.padded_xlimits[1] and
            p.lin_tdm.padded_ylimits[0] <= x[1] <= p.lin_tdm.padded_ylimits[1])


def host_trial(p, grid, max_steps, dt=None):
    """One episode of planner p driven from the host.  Returns (log, xhist, uhist, steps, status)."""
    q = p.params
    dt = float(q["dt"] if dt is None else dt)
    xh = np.full((max_steps + 1, 3), np.nan)
    uh = np.full((max_steps, 2), np.nan, dtype=np.float32)
    xh[0] = q["x0"]
    cum_obj = cum_dist = 0.0
    status = "max_steps"
    for t in range(max_steps):
        useq = p.solve()
        uh[t] = useq[0]
        xh[t + 1] = plant_step(grid, xh[t], useq[0], dt)
        p.shift_and_update(xh[t + 1], useq, num_shifts=1)
        d = np.linalg.norm(xh[t + 1, :2] - q["xgoal"]) - q["goal_tolerance"]
        cum_obj += dt + d
        cum_dist += d
        if d <= 0:
            status = "goal"
            break
        if not within(p, xh[t + 1]):            # the next solve() would refuse
            status = "left_map"
            break
    n = t + 1
    reached = status == "goal"
    if not reached:
        cum_obj += d / q["v_post_rollout"]
    log = dict(time_to_goal=n * dt if reached else np.nan, success=reached, dist_to_goal=np.nan if reached else d,
               cum_dist_to_goal=cum_dist, avg_dist_to_goal=cum_dist / n, cum_obj=cum_obj)
    return log, xh, uh, n, status
