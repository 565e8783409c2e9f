"""Host restatement of the barebone notebook's closed loop (TEST INFRASTRUCTURE): the episode
MPPI_Batch.run_barebone_trials runs on the device, written out step by step in numpy -- solve, the nominal unicycle step
in float64, shift_and_update, stop once within goal_tolerance -- plus the obstacle-contact rule and the trial-log
conventions.  Used by the tests and bench_trials.py as the reference the device episode must reproduce."""
import numpy as np


def plant_step(x, u, dt):
    """The notebook's step (cell 7) from pose x (float64 (3,)) with control u (float32 (2,)), all in float64.  The
    controls are widened first: NumPy 1 evaluated the notebook's ``cfg.dt*u_curr[1]`` in float64, while NumPy 2's
    scalar promotion would round that product to float32."""
    v, w = float(u[0]), float(u[1])
    xn = np.empty(3)
    xn[0] = x[0] + dt * np.cos(x[2]) * v
    xn[1] = x[1] + dt * np.sin(x[2]) * v
    xn[2] = x[2] + dt * w
    return xn


def obstacles(p):
    """The planner's obstacles as the engine stores them: float32 (n, 3) rows x, y, radius."""
    q = p.params
    if "obstacle_positions" not in q or not len(q["obstacle_positions"]):
        return np.zeros((0, 3), dtype=np.float32)
    pos = np.asarray(q["obstacle_positions"]).astype(np.float32).reshape(-1, 2)
    rad = np.asarray(q["obstacle_radius"]).astype(np.float32).reshape(-1)
    return np.concatenate([pos, rad[:, None]], 1)


def in_contact(x, obs):
    """Pose x touches an obstacle: (x - ox)**2 + (y - oy)**2 <= r**2 in float64 from the float32 obstacle, every
    operation rounded on its own (the rollout's rule: only a positive difference is outside)."""
    for ox, oy, r in np.asarray(obs, dtype=np.float32).astype(np.float64):
        ex, ey = x[0] - ox, x[1] - oy
        if ex * ex + ey * ey <= r * r:
            return True
    return False


def goal_distance(p, x):
    q = p.params
    xg = np.asarray(q["xgoal"], dtype=np.float64)
    dx, dy = x[0] - xg[0], x[1] - xg[1]
    return np.sqrt(dx * dx + dy * dy) - float(q["goal_tolerance"])


def host_trial(p, max_steps, dt=None, solve=None):
    """One episode of planner p driven from the host (u = solve(p), default p.solve()).  Returns
    (log, xhist, uhist, steps, status, contact_steps)."""
    q = p.params
    dt = float(q["dt"] if dt is None else dt)
    obs = obstacles(p)
    xh = np.full((max_steps + 1, 3), np.nan)
    uh = np.full((max_steps, 2), np.nan, dtype=np.float32)
    xh[0] = q["x0"]
    cum_dist, contacts = 0.0, 0
    status = "max_steps"
    for t in range(max_steps):
        useq = p.solve() if solve is None else solve(p)
        uh[t] = useq[0]
        xh[t + 1] = plant_step(xh[t], useq[0], dt)
        p.shift_and_update(xh[t + 1], useq, num_shifts=1)
        contacts += in_contact(xh[t + 1], obs)
        d = goal_distance(p, xh[t + 1])
        cum_dist += d
        if d <= 0:
            status = "goal"
            break
    n = t + 1
    reached = status == "goal"
    log = dict(time_to_goal=n * dt if reached else np.nan, success=reached, dist_to_goal=np.nan if reached else d,
               cum_dist_to_goal=cum_dist, avg_dist_to_goal=cum_dist / n, contact_steps=contacts)
    return log, xh, uh, n, status, contacts
