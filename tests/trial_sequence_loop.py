"""Host restatement of the trial-sequence loop (TEST INFRASTRUCTURE): the episodes MPPI_Batch.run_trial_sequences runs
on the device, written out step by step in numpy on the host -- per ground-truth grid one episode of the benchmark's
trial() (tests/trial_loop.py: plant step, stop rules and log conventions) on the same planner, its plant started at
params['x0'] of the call.  Used by the GPU tests as the reference the device sequences must reproduce."""
import numpy as np

from tests.trial_loop import plant_step, within


def host_episode(p, grid, max_steps, x_start, dt=None):
    """One episode of planner p driven from the host with its plant started at x_start; the first solve plans from
    whatever params['x0'] holds.  Returns (log, xhist, uhist, steps, status) as tests/trial_loop.host_trial."""
    q = p.params
    dt = float(q["dt"] if dt is None else dt)
    xh = np.full((max_steps + 1, 3), np.nan)
    uh = np.full((max_steps, 2), np.nan, dtype=np.float32)
    xh[0] = x_start
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


def host_sequence(p, grids, max_steps, dt=None, reset_x0=False):
    """The episodes of MPPI_Batch.run_trial_sequences for planner p driven from the host: one host_episode per grid on
    the same planner, each plant started at params['x0'] of the call.  reset_x0: params['x0'] set back to that start
    before every episode; else an episode plans its first solve from the previous one's final pose, and one that left
    the map ends the sequence.  Returns a list of host_episode tuples, None for an episode that did not run."""
    x_start = np.array(p.params["x0"], dtype=np.float64)
    out = []
    for g in grids:
        if reset_x0:
            p.params["x0"] = x_start.copy()
        elif out and (out[-1] is None or out[-1][4] == "left_map"):
            out.append(None)
            continue
        out.append(host_episode(p, g, max_steps, x_start, dt))
    return out
