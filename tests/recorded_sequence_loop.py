"""Host restatement of a recorded trial sequence (TEST INFRASTRUCTURE): the loop of
tests/trial_sequence_loop.host_sequence with get_state_rollout() at each episode's own steps t with t % n == 0, after
the step's solve and plant step and before shift_and_update -- what run_trial_sequences(..., record_every=n) records on
the device.  Either the numpy plant step drives it (an independent reference), or the device's trajectory is replayed
(``replay``), which makes every solve, record and the planner's final state comparable bit for bit."""
import numpy as np

from tests.trial_loop import plant_step, within


def recorded_episode(p, grid, max_steps, every, x_start, dt=None, solve=None, replay=None):
    """One episode of planner p with its plant started at x_start; the first solve plans from whatever params['x0']
    holds.  ``solve(p)`` (default p.solve()) gives the control sequence.  ``replay`` = (xhist (max_steps+1, 3), steps):
    the episode steps to those poses and runs those steps; else the numpy plant step and run_trials' stop rules.
    Returns (xhist, uhist, steps, status, records): records float32 (R, V, T+1, 3), R = ceil(max_steps / every), record
    r from step r * every, NaN from ceil(steps / every) on; status None when replayed."""
    q = p.params
    dt = float(q["dt"] if dt is None else dt)
    R = -(-max_steps // every)
    recs = np.full((R, int(p.num_vis_state_rollouts), p.num_steps + 1, 3), np.nan, dtype=np.float32)
    xh = np.full((max_steps + 1, 3), np.nan)
    uh = np.full((max_steps, 2), np.nan, dtype=np.float32)
    xh[0] = x_start
    status = None
    last = replay[1] if replay is not None else max_steps
    for t in range(last):
        useq = (solve or (lambda pl: pl.solve()))(p)
        uh[t] = useq[0]
        xh[t + 1] = replay[0][t + 1] if replay is not None else plant_step(grid, xh[t], useq[0], dt)
        if t % every == 0:
            recs[t // every] = p.get_state_rollout()
        p.shift_and_update(xh[t + 1], useq, num_shifts=1)
        if replay is not None:
            continue
        d = np.linalg.norm(xh[t + 1, :2] - q["xgoal"]) - q["goal_tolerance"]
        status = "goal" if d <= 0 else "left_map" if not within(p, xh[t + 1]) else None
        if status:
            break
    n = t + 1
    if replay is None and status is None:
        status = "max_steps"
    return xh, uh, n, status, recs


def recorded_sequence(p, grids, max_steps, every, dt=None, reset_x0=False, solve=None, replay=None):
    """The recorded episodes of run_trial_sequences for planner p: one recorded_episode per grid, each plant started at
    params['x0'] of the call; reset_x0 and the left_map rule as in host_sequence.  ``replay`` = (xhist (E, max_steps+1,
    3), steps (E,), episodes run) of the device's output for p.  Returns a list of recorded_episode tuples, None for an
    episode that did not run."""
    x_start = np.array(p.params["x0"], dtype=np.float64)
    out = []
    for e, g in enumerate(grids):
        if reset_x0:
            p.params["x0"] = x_start.copy()
        if replay is not None and e >= replay[2]:
            out.append(None)
            continue
        if replay is None and not reset_x0 and out and (out[-1] is None or out[-1][3] == "left_map"):
            out.append(None)
            continue
        rp = None if replay is None else (replay[0][e], int(replay[1][e]))
        out.append(recorded_episode(p, g, max_steps, every, x_start, dt, solve, rp))
    return out
