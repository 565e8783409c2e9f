"""``MPPI_Batch`` -- K independent one-map planners solved together, one kernel launch per stage for the whole batch.

    from mppi_numba_b200 import MPPI_Batch
    batch = MPPI_Batch([planner_0, planner_1, ...])     # MPPI_Numba (use_det_dynamics or
                                                         # use_nom_dynamics_with_speed_map) or barebone.MPPI_Numba
    u = batch.solve()                                    # np.float32 (K, T, 2) == [p.solve() for p in planners]
    for k, p in enumerate(planners):
        p.shift_and_update(new_x0[k], u[k])             # the per-planner closed-loop calls stay as they are

Each planner keeps its own params, TDMs, warm start and RNG streams; ``solve()`` leaves every one of them exactly as
``planner.solve()`` called on planners[0], planners[1], ... in that order would (include/b200mppi.h, batched one-map
solves).  The planners must share N, T, the device and the mode; their TDMs must not be shared between planners.

``MPPI_StochasticBatch(planners)`` does the same for use_tdm (CVaR-cost) planners of equal N, T and
num_grid_samples (any M a use_tdm planner takes, up to 15000 through Config): one launch per stage for noise, rollout,
CVaR and update, the map sampling per planner (include/b200mppi.h, batched stochastic solves).

``run_trials(traction_grids, max_steps)`` runs the benchmark's closed-loop episode (solve, plant step on a ground-truth
``TractionGrid``, shift_and_update, stop at the goal) for every det-dynamics or speed-map planner at once on the GPU,
without a host round trip per step (include/b200mppi.h, closed-loop trials); ``MPPI_StochasticBatch.
run_stochastic_trials`` does the same for use_tdm planners.  ``run_barebone_trials(max_steps)`` runs the barebone
notebook's closed loop (nominal unicycle, no map) for barebone planners and counts the steps that end in an obstacle.

``run_trial_sequences(traction_grids, max_steps)`` runs several such episodes per planner back to back, on the same
planners and without a reset in between, as the reference benchmark runs its trials per environment.

``get_state_rollout()`` is every planner's get_state_rollout() with one launch, and ``record_every=n`` on any trial call
records those rollouts at every n-th step inside the episodes, as the notebooks' drawing loop calls it.

Every trial call takes ``DeviceTractionGrid`` realisations (``draw_traction_grids``) wherever it takes a
``TractionGrid``: the plant reads them in GPU memory, with no upload, and the results are those of the same grids on
the host.

``share_tdms=True`` lets planners share a lin/ang TDM pair (many robots on one map, or one environment solved at several
cvar_alpha): each shared pair is sampled once per call, and each planner ends as its own call on a private copy of the
pair would leave it (include/b200mppi.h, planners sharing TDM pairs).

``MPPI_MixedBatch(planners)`` holds det-dynamics, speed-map and use_tdm planners together -- the methods the reference
benchmark compares -- and runs their solves, trials and trial sequences in one call each, every planner ending as the
batch of its own kind would leave it (include/b200mppi.h, mixed batches).

``device_loop()`` opens a ``DeviceLoop`` on any of these batches: the receding-horizon loop with the caller's own plant
(a simulator, a learned model, a state estimate in GPU memory), whose ``solve()`` and ``shift_and_update(x)`` run on the
batch's stream with no host wait (include/b200mppi.h, device loops).
"""
import ctypes as C
import sys

import numpy as np

from . import _lib
from ._lib import DeviceArray, check, lib, ptr
from .terrain import DeviceTractionGrid

TRIAL_STATUS = {_lib.TRIAL_GOAL: "goal", _lib.TRIAL_MAX_STEPS: "max_steps", _lib.TRIAL_LEFT_MAP: "left_map",
                _lib.TRIAL_NOT_RUN: "not_run"}


def _kind(p):
    """('barebone' | 'det' | 'spd' | 'tdm', world_size) of a planner object."""
    from .barebone import MPPI_Numba as Barebone
    if isinstance(p, Barebone):
        return "barebone", 1
    if getattr(p, "use_tdm", False):
        return "tdm", p.world_size
    if getattr(p, "use_det_dynamics", False):
        return "det", p.world_size
    if getattr(p, "use_nom_dynamics_with_speed_map", False):
        return "spd", p.world_size
    return "other", getattr(p, "world_size", 1)


class MPPI_Batch(object):
    """Borrows ``planners`` (keeps them alive) and solves them with one launch per stage.  ``share_tdms=True``: planners
    with the same (lin_tdm, ang_tdm) objects form a group whose pair is sampled once per call (see ``solve``)."""

    def __init__(self, planners, share_tdms=False):
        planners = list(planners)
        if not planners:
            raise ValueError("MPPI_Batch: no planners")
        kinds = [_kind(p) for p in planners]
        for i, (kind, ws) in enumerate(kinds):
            if kind == "tdm":
                raise ValueError("MPPI_Batch: planner %d uses use_tdm: the stochastic mode is not batched" % i)
            if kind == "other":
                raise ValueError("MPPI_Batch: planner %d is neither a det-dynamics, speed-map nor barebone planner" % i)
            if ws != 1:
                raise ValueError("MPPI_Batch: planner %d has world_size %d (a batch holds single-rank planners)" % (i, ws))
            if kind != kinds[0][0]:
                raise ValueError("MPPI_Batch: planner %d is a %s planner, planner 0 a %s planner (kinds cannot be mixed)"
                                 % (i, kind, kinds[0][0]))
        self._create(planners, kinds[0][0], lib.b200mppi_batch_create, share_tdms)

    def _create(self, planners, kind, create, share_tdms):
        """Borrow ``planners`` and create the batch's handle with the C constructor ``create``; ``share_tdms``: turn
        TDM sharing on."""
        self.planners = planners
        self.kind = kind
        self.order = list(range(len(planners)))        # the caller's index of each planner, named in refusals
        self._tdm = [_kind(p)[0] == "tdm" for p in planners]
        self.num_steps = planners[0].num_steps
        self.share_tdms = bool(share_tdms)
        self._handle = None
        self._loop = None                              # the open DeviceLoop
        handles = (C.c_void_p * len(planners))(*[p._handle.value for p in planners])
        h = C.c_void_p()
        check(create(handles, len(planners), C.byref(h)))
        self._handle = h
        if self.share_tdms:
            check(lib.b200mppi_batch_share_tdms(self._handle, 1))

    def _check_groups(self, name):
        """With share_tdms: the overlaps between planners' TDMs that sharing refuses (a TDM that is lin_tdm of one
        planner and ang_tdm of another, lin shared but not ang or the reverse, unequal alpha_dyn on one stochastic
        pair), as ValueError naming both planners, before any work is issued.  The library refuses the same."""
        if not self.share_tdms or self.kind == "barebone":
            return
        for i, p in enumerate(self.planners):
            for j, q in enumerate(self.planners[:i]):
                both = "%s: planners %d and %d" % ((name,) + tuple(sorted((self.order[j], self.order[i]))))
                if p.lin_tdm is q.ang_tdm or p.ang_tdm is q.lin_tdm:
                    raise ValueError(both + ": a TDM is lin_tdm of one and ang_tdm of the other (a shared TDM pair "
                                     "must be the same (lin_tdm, ang_tdm) of every planner on it)")
                if (p.lin_tdm is q.lin_tdm) != (p.ang_tdm is q.ang_tdm):
                    raise ValueError(both + " share %s (a shared TDM pair must be the same (lin_tdm, ang_tdm) of every "
                                     "planner on it)" % ("lin_tdm but not ang_tdm" if p.lin_tdm is q.lin_tdm
                                                         else "ang_tdm but not lin_tdm"))
                if self._tdm[i] and p.lin_tdm is q.lin_tdm:
                    a, b = float(q.params.get("alpha_dyn", 1.0)), float(p.params.get("alpha_dyn", 1.0))
                    if a != b:
                        raise ValueError(both + " share a TDM pair but have alpha_dyn %r and %r (a shared pair is "
                                         "sampled once, at one alpha_dyn)" % (a, b))

    def __del__(self):
        h, self._handle = getattr(self, "_handle", None), None
        if h:
            try:
                lib.b200mppi_batch_destroy(h)
            except Exception:
                pass

    def _refuse_in_loop(self, name):
        """ValueError while a device loop is open on the batch."""
        if self._loop is not None:
            raise ValueError("%s: a device loop is open on this batch (close it first)" % name)

    def device_loop(self, max_obstacles=0):
        """Open a ``DeviceLoop`` on the batch: ``solve()``, ``shift_and_update(x)``, ``set_goals(g)`` and (barebone)
        ``set_obstacles(obs)`` enqueued on the batch's stream, in GPU memory, for a plant of the caller's own (see
        DeviceLoop).  ``max_obstacles``: a barebone loop's obstacle capacity per planner, at least the largest obstacle
        count of its planners."""
        return DeviceLoop(self, max_obstacles)

    def __len__(self):
        return len(self.planners)

    def solve(self):
        """One solve() of every planner.  Returns np.float32 (K, T, 2), or None (with the planner's index and the
        reason printed) when a planner's preconditions fail -- then nothing is solved.
        With share_tdms, each shared TDM pair is sampled once, and every planner (u, u_prev_d alias, noise, costs,
        weights, RNG streams) ends exactly as after its own solve() on a private copy of its pair taken before the
        call; the shared TDMs end as every copy.  Raises ValueError (naming both planners) before any work for the
        overlaps sharing refuses."""
        u = self._solve("MPPI_Batch")
        if u is not None:
            for p in self.planners:                    # as each planner's own solve() does (mppi.py:292,362)
                p.u_prev_d = p._u_prev_buf
        return u

    def _solve(self, name):
        self._refuse_in_loop(name)
        for i, p in enumerate(self.planners):
            if not p.check_solve_conditions():
                print("{}: planner {}: MPPI solve condition not met. Cannot solve. Return".format(name, self.order[i]))
                return None
        self._check_groups(name)
        for p in self.planners:
            p.move_mppi_task_vars_to_device()          # each planner's params POD (and TDMs / obstacles)
        u = np.empty((len(self.planners), self.num_steps, 2), dtype=np.float32)
        check(lib.b200mppi_batch_solve(self._handle, ptr(u)))
        return u

    def set_stream(self, cuda_stream):
        """Issue the batch's work on ``cuda_stream`` (a raw cudaStream_t as int, e.g. torch's ``stream.cuda_stream``)."""
        self._refuse_in_loop("%s.set_stream" % type(self).__name__)
        check(lib.b200mppi_batch_set_stream(self._handle, C.c_void_p(int(cuda_stream))))

    def launch_count(self):
        """Kernel launches issued by this batch since it was created."""
        n = C.c_int64()
        check(lib.b200mppi_batch_launch_count(self._handle, C.byref(n)))
        return int(n.value)

    def get_state_rollout(self):
        """Every planner's get_state_rollout() with one launch: np.float32 (K, V, T+1, 3), the state sequences of each
        planner's current optimal controls (over its first V sampled maps for use_tdm planners; for the others the
        optimal sequence plus V-1 noisy samples).  Afterwards every planner, its state_rollout_batch_d included, is as
        after planners[0].get_state_rollout(), planners[1].get_state_rollout(), ...  Raises ValueError (naming the
        planner) when a planner's params are not set or the planners' num_vis_state_rollouts differ; nothing is issued
        then."""
        self._refuse_in_loop("%s.get_state_rollout" % type(self).__name__)
        V = self._vis_count("MPPI_Batch.get_state_rollout")
        for i, p in enumerate(self.planners):
            if not p.params_set:
                raise ValueError("MPPI_Batch.get_state_rollout: planner %d: MPPI parameters are not set" % self.order[i])
        for p in self.planners:
            p.move_mppi_task_vars_to_device()
        out = np.empty((len(self.planners), V, self.num_steps + 1, 3), dtype=np.float32)
        check(lib.b200mppi_batch_get_state_rollout(self._handle, ptr(out), out.nbytes))
        return out

    def _vis_count(self, name):
        """V of the batch's visualisation rollouts: every planner's num_vis_state_rollouts, which must be equal."""
        V = int(self.planners[0].num_vis_state_rollouts)
        for i, p in enumerate(self.planners):
            if int(p.num_vis_state_rollouts) != V:
                raise ValueError("%s: planner %d has num_vis_state_rollouts %d, planner %d %d (V must be equal)"
                                 % (name, self.order[i], int(p.num_vis_state_rollouts), self.order[0], V))
        return V


    def run_trials(self, traction_grids, max_steps, dt=None, record_every=None):
        """One closed-loop episode per planner, on the GPU: up to ``max_steps`` rounds of ``u = solve()``, a plant step
        on ``traction_grids[k]`` (a ``TractionGrid``, float or ``use_int8``, or a ``DeviceTractionGrid``) with
        ``u[0]`` and ``shift_and_update``, stopping once the planner is within ``goal_tolerance`` of its goal -- the
        loop of the benchmark's ``trial()``, whose ``dt`` argument (default: each planner's ``params['dt']``) is used as
        a float64.  A planner also stops when its pose leaves the padded map limits, where its next ``solve()`` would
        be refused.

        Afterwards every planner (controls, noise, costs, weights, RNG streams, its TDMs' streams and sampled maps, and
        ``params['x0']``) is exactly as after that host loop.  With share_tdms, a shared pair is sampled once per step
        while any of its planners runs: every planner ends as after its own episode on a private copy of its pair
        (histories, logs and records included), and the shared TDMs as the copy of the longest-running planner.
        Returns a dict:
          ``logs``: per planner, the trial log of ``trial()`` (time_to_goal, success, dist_to_goal, cum_dist_to_goal,
                    avg_dist_to_goal, cum_obj) with its NaN conventions; a planner that left the map is logged as one
                    that did not reach its goal;
          ``xhist`` float64 (K, max_steps+1, 3) and ``uhist`` float32 (K, max_steps, 2), NaN after a planner's last
          step; ``steps`` (K,) int; ``status`` (K,) of "goal" | "max_steps" | "left_map".
        ``record_every=n`` also records the visualisation rollouts of every step ``s`` with ``s % n == 0``, what
        ``get_state_rollout()`` called after the plant step and before ``shift_and_update`` returns (the notebooks'
        ``t % plot_every_n == 0``), and the dict gains ``state_rollouts`` float32 (K, R, V, T+1, 3), R =
        ceil(max_steps / n), whose record r belongs to step ``rollout_steps[r]`` = r n and is NaN from the planner's
        ``steps`` on, and ``rollout_steps`` (R,).  Everything else is as without recording, and each planner's
        state_rollout_batch_d holds its last record.
        Raises ValueError (naming the planner) for barebone batches, a grid count other than K, max_steps < 1,
        num_opt < 1, a grid of another dtype than float64 or integer, a planner that cannot solve (e.g. its start
        pose is outside the padded map limits), record_every < 1 and unequal num_vis_state_rollouts; B200MPPIError
        when a planner's TDM pair cannot be sampled by the batched sampler (its lin and ang streams diverged, or its
        PMF is not one the staged sampler takes); with share_tdms, ValueError for the overlaps sharing refuses.  Nothing
        is issued when the call is refused.
        The planners' maps may differ in size, resolution and bin count: each step samples the maps with one launch
        per class of pairs sharing the padded bin count and thread tile, so a batch on one map geometry issues the
        launches it always did."""
        if self.kind not in ("det", "spd"):
            raise ValueError("MPPI_Batch.run_trials: planner 0 is a %s planner (trials need det-dynamics or speed-map "
                             "planners)" % self.kind)
        return self._trials("MPPI_Batch.run_trials", lib.b200mppi_batch_run_trials, traction_grids, max_steps, dt,
                            record_every, _lib.TRIALS_MAP)

    def run_barebone_trials(self, max_steps, dt=None, record_every=None):
        """The barebone notebook's closed loop for every planner at once, on the GPU: up to ``max_steps`` rounds of
        ``u = solve()``, a nominal unicycle step with ``u[0]`` in float64 (``dt`` as a float64, default: each planner's
        ``params['dt']``) and ``shift_and_update``, stopping once the planner is within ``goal_tolerance`` of its goal.
        Each step's new pose is checked against the planner's obstacles: it touches one when
        ``(x - ox)**2 + (y - oy)**2 <= r**2`` in float64, the rollout's rule.  Contacts are counted; they do not stop
        the episode.

        Afterwards every planner (controls, u_prev_d alias, noise, costs, weights, RNG streams and ``params['x0']``) is
        exactly as after that host loop.  Returns a dict:
          ``logs``: per planner, time_to_goal, success, dist_to_goal, cum_dist_to_goal and avg_dist_to_goal with
                    run_trials' NaN conventions, and contact_steps (barebone params have no v_post_rollout, so there
                    is no cum_obj);
          ``xhist`` float64 (K, max_steps+1, 3) and ``uhist`` float32 (K, max_steps, 2), NaN after a planner's last
          step; ``steps`` (K,) int; ``status`` (K,) of "goal" | "max_steps"; ``contact_steps`` (K,) int, the steps
          whose new pose touched an obstacle.  ``record_every`` as in run_trials.
        Raises ValueError (naming the planner) for other batches, max_steps < 1, num_opt < 1, a planner that cannot
        solve, a non-finite x0, xgoal or goal_tolerance, a dt that is not finite and positive, record_every < 1 and
        unequal num_vis_state_rollouts.  Nothing is issued when the call is refused."""
        if self.kind != "barebone":
            raise ValueError("MPPI_Batch.run_barebone_trials: planner 0 is a %s planner (barebone trials run barebone "
                             "planners; run_trials runs det-dynamics and speed-map planners)" % self.kind)
        return self._trials("MPPI_Batch.run_barebone_trials", lib.b200mppi_batch_run_barebone_trials, None, max_steps,
                            dt, record_every, _lib.TRIALS_BAREBONE)

    def _trial_descs(self, name, seqs, max_steps, dt, record_every, episodes):
        """The checks every trial call makes before its C entry point (max_steps, record_every, V, the TDM groups, and
        each planner's solve conditions and num_opt), and the trial descriptors of ``seqs`` (per planner its grids, one
        per episode; None for barebone) planner-major, the refusals naming the episode when ``episodes``.  Returns
        (max_steps, record_every, V, descs, first, keep): planner i's descriptors are descs[first[i]:first[i + 1]], and
        ``keep`` holds what they point to."""
        self._refuse_in_loop(name)
        max_steps = int(max_steps)
        if max_steps < 1:
            raise ValueError("%s: max_steps %d < 1" % (name, max_steps))
        V = None
        if record_every is not None:
            record_every = int(record_every)
            if record_every < 1:
                raise ValueError("%s: record_every %d < 1" % (name, record_every))
            V = self._vis_count(name)
        self._check_groups(name)
        first = np.concatenate([[0], np.cumsum([len(g) for g in seqs], dtype=np.int64)])
        descs = (_lib.TrialDesc * int(first[-1]))()
        keep = []
        for i, p in enumerate(self.planners):
            who = "%s: planner %d" % (name, self.order[i])
            if not p.check_solve_conditions():
                raise ValueError("%s cannot solve (reason printed above)" % who)
            if int(p.params["num_opt"]) < 1:
                raise ValueError("%s has num_opt %d < 1" % (who, int(p.params["num_opt"])))
            for e, g in enumerate(seqs[i]):
                _fill_desc(who + (", episode %d" % e if episodes else ""), p, g, dt, descs[first[i] + e], keep)
        for p in self.planners:
            p.move_mppi_task_vars_to_device()
        return max_steps, record_every, V, descs, first, keep

    def _trials(self, name, entry, traction_grids, max_steps, dt, record_every, kind):
        """The marshalling of a closed-loop trial call through the C entry point ``entry`` (with record_every set:
        b200mppi_batch_run_trials_recorded with trial kind ``kind``) and the logs built from its results (run_trials,
        run_barebone_trials with traction_grids None, MPPI_StochasticBatch.run_stochastic_trials); ``name`` prefixes
        the refusals."""
        K = len(self.planners)
        barebone = traction_grids is None
        grids = [None] * K if barebone else list(traction_grids)
        if len(grids) != K:
            raise ValueError("%s: %d traction grids for %d planners" % (name, len(grids), K))
        max_steps, record_every, V, descs, _, keep = self._trial_descs(name, [[g] for g in grids], max_steps, dt,
                                                                        record_every, False)
        xhist = np.empty((K, max_steps + 1, 3), dtype=np.float64)
        uhist = np.empty((K, max_steps, 2), dtype=np.float32)
        res = (_lib.TrialResult * K)()
        issued = C.c_int32()
        contacts = np.zeros(K, dtype=np.int32)
        if record_every is None:
            outs = (ptr(xhist), ptr(uhist), res) + ((ptr(contacts),) if barebone else ())
            check(entry(self._handle, descs, max_steps, *outs, C.byref(issued)))
        else:
            R = -(-max_steps // record_every)
            rollouts = np.empty((K, R, V, self.num_steps + 1, 3), dtype=np.float32)
            check(lib.b200mppi_batch_run_trials_recorded(self._handle, kind, descs, max_steps, ptr(xhist), ptr(uhist),
                                                         res, ptr(contacts) if barebone else None, record_every,
                                                         ptr(rollouts), rollouts.nbytes, C.byref(issued)))
        self.steps_issued = int(issued.value)
        steps = np.array([r.steps for r in res], dtype=np.int64)
        status = [TRIAL_STATUS[r.status] for r in res]
        logs = []
        for i, p in enumerate(self.planners):
            if not self._tdm[i]:
                p.u_prev_d = p._u_prev_buf             # as each planner's own solve() does (mppi.py:292,362)
            p.params["x0"] = xhist[i, steps[i]].copy()  # shift_and_update(x_next, ...)
            log = _trial_log(res[i], descs[i], barebone)
            if barebone:
                log["contact_steps"] = int(contacts[i])
            logs.append(log)
        out = dict(logs=logs, xhist=xhist, uhist=uhist, steps=steps, status=status)
        if barebone:
            out["contact_steps"] = contacts.astype(np.int64)
        if record_every is not None:
            out["state_rollouts"] = rollouts
            out["rollout_steps"] = np.arange(R, dtype=np.int64) * record_every
        return out


    def run_trial_sequences(self, traction_grids, max_steps, dt=None, reset_x0=False, record_every=None):
        """Several closed-loop episodes per planner, back to back on the GPU: planner k runs one episode of
        ``run_trials`` (``run_stochastic_trials`` for use_tdm planners) on each grid (``TractionGrid`` or
        ``DeviceTractionGrid``) of the non-empty list ``traction_grids[k]`` in turn, each starting its plant at
        ``x_start = params['x0']`` of the call, with the stop rules, ``dt`` and log conventions of run_trials.
        Between episodes nothing is reset: the planner keeps its warm start, RNG streams and its TDMs' streams and maps
        -- the loop the reference benchmark runs over trials_per_env realisations after one setup().
          ``reset_x0=False`` (the benchmark's loop): ``params['x0']`` is left at the previous episode's final pose, so
              an episode's first solve plans from there.  An episode ending "left_map" ends the planner's sequence
              (its next solve would be refused); the later episodes are "not_run".
          ``reset_x0=True``: ``params['x0'] = x_start`` before every episode, as a user resetting it would; every
              episode runs.
        Afterwards every planner is exactly as after that host loop over its run episodes (buffers, RNG streams, its
        TDMs' streams and sampled maps, ``sample_box()``), ``params['x0']`` the final pose of its last run episode.  With
        share_tdms a shared pair ends as the copy of the member that ran the most steps in all.  Episodes cost no extra
        launch: the batch runs until every planner's sequence has ended.
        Returns a dict: ``logs``, K lists of E_k trial logs (None for an episode that did not run); ``xhist`` float64
        (K, Emax, max_steps+1, 3) and ``uhist`` float32 (K, Emax, max_steps, 2), NaN wherever nothing ran; ``steps``
        (K, Emax) int, 0 where nothing ran; ``status``, K lists of E_k of "goal" | "max_steps" | "left_map" |
        "not_run"; ``episodes_run`` (K,) int.  ``steps_issued`` is set as run_trials sets it.
        ``record_every=n`` records, in each run episode at each of its own steps ``t`` with ``t % n == 0``, what
        run_trials records there (``get_state_rollout()`` after the step's solve and plant step, before
        ``shift_and_update``); the dict gains ``state_rollouts`` float32 (K, Emax, R, V, T+1, 3), R = ceil(max_steps / n),
        NaN after an episode's last step and everywhere for an episode that did not run or does not exist, and
        ``rollout_steps`` (R,) = r n, steps of the episode.  Each planner's state_rollout_batch_d ends with the last
        record of its last run episode; everything else is as without recording.  Which planners record at a step is
        decided on the device, so a recorded sequence issues the record launches at every step: 1 + C2 per step more
        than without recording (C2: the stochastic sampler launch classes, 0 for a batch without use_tdm planners).
        Raises ValueError for barebone batches (run_barebone_trial_sequences runs them), a list count other than K, an
        empty list, record_every < 1, unequal num_vis_state_rollouts when recording, and whatever run_trials refuses
        for any of the grids; nothing is issued then."""
        name = "%s.run_trial_sequences" % type(self).__name__
        if self.kind == "barebone":
            raise ValueError("%s: planner 0 is a barebone planner (trial sequences run det-dynamics, speed-map and "
                             "use_tdm planners)" % name)
        K = len(self.planners)
        seqs = [list(g) for g in traction_grids]
        if len(seqs) != K:
            raise ValueError("%s: %d lists of traction grids for %d planners" % (name, len(seqs), K))
        for i, g in enumerate(seqs):
            if not g:
                raise ValueError("%s: planner %d: empty list of traction grids" % (name, self.order[i]))
        kind = {"tdm": _lib.TRIALS_STOCHASTIC, "mixed": _lib.TRIALS_MIXED}.get(self.kind, _lib.TRIALS_MAP)
        return self._sequences(name, seqs, max_steps, dt, reset_x0, record_every, kind)

    def run_barebone_trial_sequences(self, episodes, max_steps, dt=None, reset_x0=False, record_every=None):
        """Several episodes of run_barebone_trials per planner, back to back on the GPU: planner k runs ``episodes``
        (an int, or K ints each >= 1) episodes of the barebone notebook's loop, each starting its plant at
        ``x_start = params['x0']`` of the call.  Between episodes the planner keeps its warm start and RNG streams;
        ``reset_x0`` as in run_trial_sequences.  A barebone plant has no map to leave, so every episode runs.
        Afterwards every planner is exactly as after that host loop (tests/barebone_trial_loop.py per episode).
        Returns run_trial_sequences' dict with barebone logs (each with its contact_steps), status "goal" |
        "max_steps", and ``contact_steps`` (K, Emax) int, per episode the steps whose new pose touched an obstacle (0
        where no episode exists); ``record_every`` as in run_trial_sequences (no completion launches: 1 per step).
        Raises ValueError (naming the planner) for other batches, an episode count other than K or < 1, and whatever
        run_barebone_trials refuses; nothing is issued then."""
        name = "%s.run_barebone_trial_sequences" % type(self).__name__
        if self.kind != "barebone":
            raise ValueError("%s: planner 0 is a %s planner (barebone trial sequences run barebone planners; "
                             "run_trial_sequences runs the others)" % (name, self.kind))
        K = len(self.planners)
        counts = [episodes] * K if np.ndim(episodes) == 0 else list(episodes)
        if len(counts) != K:
            raise ValueError("%s: %d episode counts for %d planners" % (name, len(counts), K))
        for i, e in enumerate(counts):
            if int(e) < 1:
                raise ValueError("%s: planner %d: episode count %d < 1" % (name, self.order[i], int(e)))
        return self._sequences(name, [[None] * int(e) for e in counts], max_steps, dt, reset_x0, record_every,
                               _lib.TRIALS_BAREBONE)

    def _sequences(self, name, seqs, max_steps, dt, reset_x0, record_every, kind):
        """The marshalling of a trial-sequence call (``seqs``: per planner its grids, None for barebone episodes) through
        b200mppi_batch_run_trial_sequences, or b200mppi_batch_run_trial_sequences_ex when recording or barebone, and
        the dict built from its per-slot results; ``name`` prefixes the refusals."""
        K = len(self.planners)
        barebone = kind == _lib.TRIALS_BAREBONE
        max_steps, record_every, V, descs, first, keep = self._trial_descs(name, seqs, max_steps, dt, record_every,
                                                                            True)
        E = np.diff(first).astype(np.int32)
        slots = int(first[-1])
        xs = np.empty((slots, max_steps + 1, 3), dtype=np.float64)
        us = np.empty((slots, max_steps, 2), dtype=np.float32)
        res = (_lib.TrialResult * slots)()
        issued = C.c_int32()
        contacts = np.zeros(slots, dtype=np.int32)
        if record_every is None and not barebone:
            check(lib.b200mppi_batch_run_trial_sequences(self._handle, kind, descs, ptr(E), max_steps,
                                                         int(bool(reset_x0)), ptr(xs), ptr(us), res, C.byref(issued)))
        else:
            if record_every is not None:                # written by the library in the returned layout
                R = -(-max_steps // record_every)
                recs = np.empty((K, int(E.max()), R, V, self.num_steps + 1, 3), dtype=np.float32)
            check(lib.b200mppi_batch_run_trial_sequences_ex(
                self._handle, kind, descs, ptr(E), max_steps, int(bool(reset_x0)), ptr(xs), ptr(us), res,
                ptr(contacts) if barebone else None, record_every or 0,
                ptr(recs) if record_every is not None else None, recs.nbytes if record_every is not None else 0,
                C.byref(issued)))
        self.steps_issued = int(issued.value)
        Emax = int(E.max())
        xhist = np.full((K, Emax, max_steps + 1, 3), np.nan)
        uhist = np.full((K, Emax, max_steps, 2), np.nan, dtype=np.float32)
        steps = np.zeros((K, Emax), dtype=np.int64)
        episodes_run = np.zeros(K, dtype=np.int64)
        logs, status = [], []
        for i, p in enumerate(self.planners):
            n = int(E[i])
            xhist[i, :n], uhist[i, :n] = xs[first[i]:first[i] + n], us[first[i]:first[i] + n]
            st = [TRIAL_STATUS[res[j].status] for j in range(first[i], first[i] + n)]
            run = sum(s != "not_run" for s in st)
            steps[i, :run] = [res[j].steps for j in range(first[i], first[i] + run)]
            logs.append([_trial_log(res[first[i] + e], descs[first[i] + e], barebone) if e < run else None
                         for e in range(n)])
            if barebone:
                for e in range(run):
                    logs[i][e]["contact_steps"] = int(contacts[first[i] + e])
            status.append(st)
            episodes_run[i] = run
            if not self._tdm[i]:
                p.u_prev_d = p._u_prev_buf             # as each planner's own solve() does (mppi.py:292,362)
            p.params["x0"] = xhist[i, run - 1, steps[i, run - 1]].copy()
        out = dict(logs=logs, xhist=xhist, uhist=uhist, steps=steps, status=status, episodes_run=episodes_run)
        if barebone:
            out["contact_steps"] = np.zeros((K, Emax), dtype=np.int64)
            for i in range(K):
                out["contact_steps"][i, :E[i]] = contacts[first[i]:first[i + 1]]
        if record_every is not None:
            out["state_rollouts"] = recs
            out["rollout_steps"] = np.arange(R, dtype=np.int64) * record_every
        return out


def _fill_desc(who, p, g, dt, d, keep):
    """Trial descriptor ``d`` of planner ``p`` on TractionGrid or DeviceTractionGrid ``g`` (None: barebone), starting
    at params['x0']; the float64 grids it points to (a device grid: the grid, which keeps its set alive) are appended
    to ``keep``.  ``who`` prefixes the refusals."""
    q = p.params
    if g is None:
        d.x0[:] = [float(v) for v in np.asarray(q["x0"], dtype=np.float64)[:3]]
        d.xgoal[:] = [float(v) for v in np.asarray(q["xgoal"], dtype=np.float64)[:2]]
        d.goal_tolerance = float(q["goal_tolerance"])
        d.dt = float(q["dt"] if dt is None else dt)
        if not np.isfinite(list(d.x0) + list(d.xgoal) + [d.goal_tolerance]).all():
            raise ValueError("%s: start pose, goal or goal_tolerance not finite" % who)
        if not (np.isfinite(d.dt) and d.dt > 0):
            raise ValueError("%s: dt %r not finite and positive" % (who, d.dt))
        return
    if isinstance(g, DeviceTractionGrid):                # read in place by the plant step
        keep.append(g)
        d.lin, d.ang = g._lin_ptr, g._ang_ptr
        d.height, d.width = g.height, g.width
    else:
        lin, ang = np.asarray(g.lin_traction), np.asarray(g.ang_traction)
        for a in (lin, ang):
            if a.dtype != np.float64 and not np.issubdtype(a.dtype, np.integer):
                raise ValueError("%s: traction grid of dtype %s (float64 or integer grids only: the plant step is "
                                 "float64)" % (who, a.dtype))
        if lin.ndim != 2 or lin.shape != ang.shape:
            raise ValueError("%s: lin / ang traction grids of shapes %s / %s" % (who, lin.shape, ang.shape))
        lin = np.ascontiguousarray(lin, dtype=np.float64)
        ang = np.ascontiguousarray(ang, dtype=np.float64)
        keep += [lin, ang]
        d.lin, d.ang = lin.ctypes.data, ang.ctypes.data
        d.height, d.width = lin.shape
    d.xlo, d.ylo, d.res = float(g.xlimits[0]), float(g.ylimits[0]), float(g.res)
    d.x0[:] = [float(v) for v in np.asarray(q["x0"], dtype=np.float64)[:3]]
    d.xgoal[:] = [float(v) for v in np.asarray(q["xgoal"], dtype=np.float64)[:2]]
    d.goal_tolerance, d.v_post_rollout = float(q["goal_tolerance"]), float(q["v_post_rollout"])
    d.dt = float(q["dt"] if dt is None else dt)
    d.pxlim[:] = [float(v) for v in p.lin_tdm.padded_xlimits]
    d.pylim[:] = [float(v) for v in p.lin_tdm.padded_ylimits]


def _trial_log(r, d, barebone):
    """The trial log of trial() from result record ``r`` of descriptor ``d``: a planner that did not reach its goal
    adds the d / v_post_rollout tail to cum_obj and has no time to goal (barebone logs have no cum_obj)."""
    n, reached = int(r.steps), r.status == _lib.TRIAL_GOAL
    cum_obj, dist = r.cum_obj, r.dist_to_goal
    if reached:
        dist = np.nan
    elif not barebone:
        cum_obj += dist / d.v_post_rollout
    log = dict(time_to_goal=n * d.dt if reached else np.nan, success=reached, dist_to_goal=dist,
               cum_dist_to_goal=r.cum_dist_to_goal, avg_dist_to_goal=r.cum_dist_to_goal / n)
    if not barebone:
        log["cum_obj"] = cum_obj
    return log


class MPPI_StochasticBatch(MPPI_Batch):
    """Borrows use_tdm ``planners`` (keeps them alive) and solves them with one launch per stage: noise, windowed
    rollout, CVaR and update; each planner's map sampling keeps its own launches.  The planners share N, T and
    num_grid_samples, which may be any M a use_tdm planner takes: above 1024 maps the one CVaR launch runs one CTA
    per control sequence instead of one warp.  ``solve()``, ``set_stream`` and ``launch_count`` as in MPPI_Batch;
    closed-loop trials through ``run_stochastic_trials``.  ``share_tdms`` as in MPPI_Batch; the planners of a shared
    pair must have equal ``alpha_dyn``."""

    def __init__(self, planners, share_tdms=False):
        planners = list(planners)
        if not planners:
            raise ValueError("MPPI_StochasticBatch: no planners")
        for i, p in enumerate(planners):
            kind, ws = _kind(p)
            if kind != "tdm":
                raise ValueError("MPPI_StochasticBatch: planner %d is a %s planner (a stochastic batch holds use_tdm "
                                 "planners; MPPI_Batch takes the others)" % (i, kind))
            if ws != 1:
                raise ValueError("MPPI_StochasticBatch: planner %d has world_size %d (a batch holds single-rank planners)"
                                 % (i, ws))
        self._create(planners, "tdm", lib.b200mppi_batch_create_stochastic, share_tdms)

    def solve(self):
        """One solve() of every planner.  Returns np.float32 (K, T, 2), or None (with the planner's index and the
        reason printed) when a planner's preconditions fail -- then nothing is solved.  u_prev_d is left alone, as a
        stochastic planner's own solve() leaves it.
        With share_tdms, each shared pair is sampled once, over the hull of its planners' reach boxes (one planner: its
        own box; whole maps if any planner's box is whole maps).  Every planner (u, noise, per-(m, n) and CVaR costs,
        weights, RNG streams) ends exactly as after its own solve() on a private copy of its pair taken before the
        call; ``sample_box()`` reports the box the pair was sampled over."""
        return self._solve("MPPI_StochasticBatch")

    def run_trials(self, traction_grids, max_steps, dt=None, record_every=None):
        raise ValueError("MPPI_StochasticBatch.run_trials: closed-loop trials run det-dynamics or speed-map batches "
                         "(a stochastic batch runs them with run_stochastic_trials)")

    def run_barebone_trials(self, max_steps, dt=None, record_every=None):
        raise ValueError("MPPI_StochasticBatch.run_barebone_trials: barebone trials run barebone batches (a stochastic "
                         "batch runs its trials with run_stochastic_trials)")

    def run_stochastic_trials(self, traction_grids, max_steps, dt=None, record_every=None):
        """MPPI_Batch.run_trials for use_tdm planners: the same arguments, episode, stop rules, returned dict and NaN
        conventions, one episode per planner on the GPU without a host round trip per step (each planner's
        map-sampling reach box is decided on the device).  Afterwards every planner is exactly as after ``steps[k]``
        rounds of ``u = batch.solve()``, the plant step on ``traction_grids[k]`` and ``shift_and_update(x_next, u[k])``:
        controls, noise, per-(m, n) and CVaR costs, weights, RNG streams, its TDMs' streams and sampled maps,
        ``sample_box()`` and ``params['x0']``.  u_prev_d is left alone, as a stochastic solve leaves it.  With
        share_tdms, a shared pair is sampled once per step over the hull of its running planners' boxes, and every
        planner ends as after its own episode on a private copy of its pair, except that ``sample_box()`` is the box
        its pair was sampled over at its last step.
        ``record_every`` as in run_trials: the records equal ``get_state_rollout()`` of that host loop, which completes
        the maps of a boxed sampling first.
        The planners' maps may differ in size, resolution and bin count, as in run_trials: each step issues one boxed
        sampler launch and one state advance per class of pairs sharing the padded bin count and thread tile.
        Raises ValueError (naming the planner) as run_trials does; B200MPPIError when a planner cannot take the windowed
        rollout, its TDM pair cannot be sampled by the batched sampler (lin == ang, diverged streams, a PMF the staged
        sampler cannot take) or a class's boxed sampler launch does not fit a CTA.  Nothing is issued when the call is
        refused."""
        return self._trials("MPPI_StochasticBatch.run_stochastic_trials", lib.b200mppi_batch_run_stochastic_trials,
                            traction_grids, max_steps, dt, record_every, _lib.TRIALS_STOCHASTIC)


class MPPI_MixedBatch(MPPI_Batch):
    """Borrows det-dynamics, speed-map and use_tdm ``planners`` (keeps them alive), in any mix and order, and runs them
    together: ``solve()``, ``run_trials``, ``run_trial_sequences``, ``get_state_rollout()``, ``launch_count()`` and
    ``set_stream`` as in MPPI_Batch, one call for all the methods of a comparison instead of one call per kind.

    Every argument and result is in the caller's planner order.  Internally the one-map planners come first, in the
    caller's order, then the use_tdm planners (``planners`` holds them so, ``order[j]`` is the caller's index of
    ``planners[j]``).  The trial calls take a ``TractionGrid`` or ``DeviceTractionGrid`` per planner (per episode) and
    return the dicts of MPPI_Batch.run_trials and run_trial_sequences.

    The contract: each planner's outputs, and the state it is left in (u, u_prev_d alias, noise, costs, weights, RNG
    streams, its TDMs' maps and generator states, ``sample_box()`` and ``params['x0']``), are bit for bit those of the
    same call on the batch of its own kind: ``MPPI_Batch`` of the det-dynamics planners, ``MPPI_Batch`` of the
    speed-map planners, ``MPPI_StochasticBatch`` of the use_tdm planners (``run_stochastic_trials`` for run_trials),
    each with the same ``share_tdms``, which groups planners exactly as those batches do.

    Raises ValueError, naming the planner(s) in the caller's order, before any work is issued: for what the batch of a
    planner's kind refuses, barebone planners (MPPI_Batch.run_barebone_trials runs them), world_size > 1, unequal
    N or T (at construction), unequal num_grid_samples among the use_tdm planners, unequal num_opt, a TDM used by
    planners of two kinds, and unequal num_vis_state_rollouts when recording or in get_state_rollout().  The library's
    own refusals raise B200MPPIError as the per-kind batches' do.  A batch of one kind issues exactly the launches of the
    batch of that kind; with both kinds a trial step at num_opt n issues 6 n + 1 + C1 + 2 C2 launches (C1, C2: the
    one-map and stochastic sampler launch classes)."""

    def __init__(self, planners, share_tdms=False):
        planners = list(planners)
        if not planners:
            raise ValueError("MPPI_MixedBatch: no planners")
        kinds = []
        for i, p in enumerate(planners):
            kind, ws = _kind(p)
            if kind == "barebone":
                raise ValueError("MPPI_MixedBatch: planner %d is a barebone planner (a mixed batch holds det-dynamics, "
                                 "speed-map and use_tdm planners; MPPI_Batch runs barebone planners)" % i)
            if kind == "other":
                raise ValueError("MPPI_MixedBatch: planner %d is neither a det-dynamics, speed-map nor use_tdm planner"
                                 % i)
            if ws != 1:
                raise ValueError("MPPI_MixedBatch: planner %d has world_size %d (a batch holds single-rank planners)"
                                 % (i, ws))
            kinds.append(kind)
        order = [i for i, k in enumerate(kinds) if k != "tdm"] + [i for i, k in enumerate(kinds) if k == "tdm"]
        for i, p in enumerate(planners):
            for what, attr in (("num_steps", "num_steps"), ("num_control_rollouts", "num_control_rollouts")):
                if getattr(p, attr) != getattr(planners[0], attr):
                    raise ValueError("MPPI_MixedBatch: planner %d has %s %d, planner 0 %d (N and T must be equal)"
                                     % (i, what, getattr(p, attr), getattr(planners[0], attr)))
        tdm = [i for i in order if kinds[i] == "tdm"]
        for i in tdm:
            if planners[i].num_grid_samples != planners[tdm[0]].num_grid_samples:
                raise ValueError("MPPI_MixedBatch: planner %d has num_grid_samples %d, planner %d %d (M must be equal)"
                                 % (i, planners[i].num_grid_samples, tdm[0], planners[tdm[0]].num_grid_samples))
        self._create([planners[i] for i in order], "mixed", lib.b200mppi_batch_create_mixed, share_tdms)
        self.order = order

    def _check_groups(self, name):
        """Equal num_opt and no TDM used by planners of two kinds, then MPPI_Batch's checks."""
        K = len(self.planners)
        for i in range(K):
            p, o = self.planners[i], self.order
            if int(p.params["num_opt"]) != int(self.planners[0].params["num_opt"]):
                raise ValueError("%s: planner %d has num_opt %d, planner %d num_opt %d (must be equal)"
                                 % (name, o[i], int(p.params["num_opt"]), o[0], int(self.planners[0].params["num_opt"])))
            for j in range(i):
                q = self.planners[j]
                if self._tdm[i] != self._tdm[j] and {id(p.lin_tdm), id(p.ang_tdm)} & {id(q.lin_tdm), id(q.ang_tdm)}:
                    a, b = sorted((o[j], o[i]))
                    raise ValueError("%s: planners %d and %d share a TDM, but one is a use_tdm planner and the other "
                                     "is not (a TDM belongs to planners of one kind)" % (name, a, b))
        super()._check_groups(name)

    def _to_caller(self, a):
        """Per-planner array or list ``a`` in the batch's order -> the caller's order."""
        if isinstance(a, np.ndarray):
            out = np.empty_like(a)
            out[self.order] = a
            return out
        out = [None] * len(a)
        for j, i in enumerate(self.order):
            out[i] = a[j]
        return out

    def _from_caller(self, a):
        """Per-planner list ``a`` in the caller's order -> the batch's order (other lengths pass through, refused as
        MPPI_Batch refuses them)."""
        a = list(a)
        return [a[i] for i in self.order] if len(a) == len(self.order) else a

    def solve(self):
        """One solve() of every planner: np.float32 (K, T, 2) in the caller's order, or None (the planner's index and
        the reason printed) when a planner's preconditions fail -- then nothing is solved."""
        u = self._solve("MPPI_MixedBatch")
        if u is None:
            return None
        for i, p in enumerate(self.planners):
            if not self._tdm[i]:
                p.u_prev_d = p._u_prev_buf             # as each one-map planner's own solve() does (mppi.py:292,362)
        return self._to_caller(u)

    def get_state_rollout(self):
        """MPPI_Batch.get_state_rollout in the caller's order: np.float32 (K, V, T+1, 3)."""
        return self._to_caller(super().get_state_rollout())

    def run_trials(self, traction_grids, max_steps, dt=None, record_every=None):
        """One closed-loop episode per planner on ``traction_grids[k]``: MPPI_Batch.run_trials for det-dynamics and
        speed-map planners, MPPI_StochasticBatch.run_stochastic_trials for use_tdm planners, with their arguments,
        returned dict (in the caller's order), ``record_every`` and refusals."""
        out = self._trials("MPPI_MixedBatch.run_trials", lib.b200mppi_batch_run_mixed_trials,
                           self._from_caller(traction_grids), max_steps, dt, record_every, _lib.TRIALS_MIXED)
        for key in ("logs", "xhist", "uhist", "steps", "status", "state_rollouts"):
            if key in out:
                out[key] = self._to_caller(out[key])
        return out

    def run_trial_sequences(self, traction_grids, max_steps, dt=None, reset_x0=False, record_every=None):
        """MPPI_Batch.run_trial_sequences for every planner, each by its kind; lists and the returned dict in the
        caller's order."""
        out = super().run_trial_sequences(self._from_caller(traction_grids), max_steps, dt, reset_x0, record_every)
        for key in ("logs", "xhist", "uhist", "steps", "status", "episodes_run", "state_rollouts"):
            if key in out:
                out[key] = self._to_caller(out[key])
        return out

    def run_barebone_trial_sequences(self, episodes, max_steps, dt=None, reset_x0=False, record_every=None):
        raise ValueError("MPPI_MixedBatch.run_barebone_trial_sequences: a mixed batch holds no barebone planners "
                         "(MPPI_Batch runs barebone trial sequences)")

    def run_barebone_trials(self, max_steps, dt=None, record_every=None):
        raise ValueError("MPPI_MixedBatch.run_barebone_trials: a mixed batch holds no barebone planners (MPPI_Batch "
                         "runs barebone trials)")


LOOP_STATUS = {_lib.LOOP_RUNNING: "running", _lib.TRIAL_LEFT_MAP: "left_map", _lib.LOOP_STOPPED: "stopped",
               _lib.LOOP_BAD_OBSTACLES: "bad_obstacles"}


class DeviceLoop(object):
    """A receding-horizon loop on a batch whose plant is the caller's, on the GPU with no host wait between calls:

        batch.set_stream(torch.cuda.current_stream().cuda_stream)    # optional; the loop runs on the batch's stream
        with batch.device_loop() as loop:
            for t in range(steps):
                u = torch.as_tensor(loop.solve(), device="cuda")       # (K, T, 2) float32, NaN rows: not solved
                x = my_plant(x, u[:, 0])                               # any GPU work on the same stream
                loop.shift_and_update(x)                               # (K, 3) float64 or float32 on the device
                loop.stop(done)                                        # optional: (K,) int32 / bool, nonzero stops k
        loop.solves, loop.shifts, loop.status                         # per planner, read at close

    Opened by ``device_loop()`` of an ``MPPI_Batch`` (det-dynamics, speed-map or barebone planners),
    ``MPPI_StochasticBatch`` or ``MPPI_MixedBatch``, with or without share_tdms.  A single planner runs in a batch of
    one.  Rows are in the caller's planner order.  Per planner the loop is the host loop of the same calls, bit for bit:
    ``loop.solve()`` is ``u = p.solve()`` (a use_tdm planner: ``MPPI_StochasticBatch([p]).solve()``) and
    ``loop.shift_and_update(x)`` is ``p.shift_and_update(x[k], u, 1)`` with ``u`` the planner's current controls (after
    a solve: that solve's).  The calls may come in any order.  Each new pose goes into the next rollout as float32(x).

    A pose outside the planner's padded map limits (float64 lo <= v <= hi; NaN fails), where its next host solve would be
    refused, stops that planner for good with status "left_map"; barebone planners have no map, so never.  ``stop(done)``
    stops planner k for good when done[k] is nonzero.  A stopped planner's rows of later ``solve()`` outputs are NaN and
    it is left untouched by every later call.

    The task can change between solves, from GPU memory, one launch per call (waypoints, a moving target, robots that
    avoid each other):

        loop.set_goals(g)                                             # (K, 2) float64 / float32 on the device
        loop.set_obstacles(obs, counts)                               # barebone: (K, O', 3) [x, y, r], counts (K,) int32

    ``set_goals(g)`` is ``p.params['xgoal'] = g[k]`` before planner k's later solves: they plan toward float32(g[k]).
    ``set_obstacles(obs, counts)`` (barebone loops only) is ``p.params['obstacle_positions'] = obs[k, :n, :2]`` and
    ``p.params['obstacle_radius'] = obs[k, :n, 2]`` with n = counts[k] (default O').  O' is at most the loop's
    ``max_obstacles``: ``device_loop(max_obstacles=O)`` sets it, and it is never below the largest obstacle count of the
    planners at open.  A count outside [0, O'], which the host's set_obstacles refuses, stops that planner for good with
    status "bad_obstacles"; its rollouts keep the last set it took.

    While the loop is open, the batch's calls and every call that reads or writes a member's state on the host
    (``solve``, ``setup`` / ``set_params``, ``shift_and_update``, ``get_state`` / ``set_state``,
    ``get_state_rollout``, the TDM setters and ``sample_grids`` of its TDMs) raise ValueError naming the planner.
    Closing (``close()``, or leaving the ``with`` block, also on an exception) waits for the stream and commits every
    planner: afterwards each is exactly as after that host loop, ``params['x0']`` the float64 value of the last pose it
    took (a float32 pose widened exactly), ``params['xgoal']``, ``params['obstacle_positions']`` and
    ``params['obstacle_radius']`` the float64 values of the last goal and obstacle set it took (a planner that took
    none keeps its own), and ``solves``, ``shifts`` (K,) int and ``status`` (K,) of "running" | "left_map" | "stopped"
    | "bad_obstacles" are set.  Launches: a solve issues what a trial step of the batch issues without its plant step,
    plus one export; ``shift_and_update``, ``stop``, ``set_goals`` and ``set_obstacles`` one each.

    CUDA graphs.  Nothing a loop call passes to the GPU changes from one call to the next (the loop counts its solves on
    the device), so a whole step, the caller's plant included, can be captured once and replayed:

        s = torch.cuda.Stream()
        batch.set_stream(s.cuda_stream)                               # before the loop opens
        u = torch.empty((K, T, 2), dtype=torch.float32, device="cuda")   # static tensors: out, pose, done
        with batch.device_loop() as loop:
            def step():
                loop.solve(out=u)
                x.copy_(my_plant(x, u[:, 0]))
                loop.stop(done_of(x, done))                           # optional: a device-computed stop
                loop.shift_and_update(x)
                goal.copy_(next_waypoint(x, goal))                    # optional: goals computed on the device
                loop.set_goals(goal)
            with torch.cuda.stream(s):
                step()                                                # warm-up: the loop's first step, eager
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g, stream=s):
                step()                                                # captured, not run
            for t in range(steps - 1):
                g.replay()                                            # stopped planners do nothing

    Replays, eager calls and more captures mix freely on one loop: each replay is the captured calls at that point of
    the loop, bit for bit.  A replay reads the arrays captured (their pointers, dtype and row stride are fixed at
    capture), so refill them in place.  ``batch.launch_count()`` counts the launches issued from the host: captured
    calls count once, replays add nothing.  While the batch's stream captures, ``close()`` raises and the loop stays
    open, and a call while torch captures on a stream other than the loop's raises ValueError before anything is
    enqueued (its launches would run at once, outside the caller's graph)."""

    def __init__(self, batch, max_obstacles=0):
        name = "%s.device_loop" % type(batch).__name__
        batch._refuse_in_loop(name)
        max_obstacles = int(max_obstacles)
        if max_obstacles < 0:
            raise ValueError("%s: max_obstacles %d < 0" % (name, max_obstacles))
        if max_obstacles > 0 and batch.kind != "barebone":
            raise ValueError("%s: max_obstacles %d for a %s batch (only barebone planners take obstacles)"
                             % (name, max_obstacles, batch.kind))
        batch._check_groups(name)
        for i, p in enumerate(batch.planners):
            who = "%s: planner %d" % (name, batch.order[i])
            if not p.check_solve_conditions():
                raise ValueError("%s cannot solve (reason printed above)" % who)
            if int(p.params["num_opt"]) < 1:
                raise ValueError("%s has num_opt %d < 1" % (who, int(p.params["num_opt"])))
        for p in batch.planners:
            p.move_mppi_task_vars_to_device()
        self.batch = batch
        self.K, self.T = len(batch.planners), batch.num_steps
        self.device = int(getattr(batch.planners[0], "device", 0))
        kind = {"barebone": _lib.TRIALS_BAREBONE, "tdm": _lib.TRIALS_STOCHASTIC,
                "mixed": _lib.TRIALS_MIXED}.get(batch.kind, _lib.TRIALS_MAP)
        limits = None
        if batch.kind != "barebone":
            limits = np.array([list(p.lin_tdm.padded_xlimits) + list(p.lin_tdm.padded_ylimits) for p in batch.planners],
                              dtype=np.float64)
        rows = np.array(batch.order, dtype=np.int32)
        h = C.c_void_p()
        lim = ptr(limits) if limits is not None else None
        if max_obstacles:
            check(lib.b200mppi_batch_loop_open_ex(batch._handle, kind, lim, ptr(rows), max_obstacles, C.byref(h)))
        else:                                          # open_ex with 0
            check(lib.b200mppi_batch_loop_open(batch._handle, kind, lim, ptr(rows), C.byref(h)))
        self._handle = h
        cap = C.c_int32()
        check(lib.b200mppi_loop_obstacle_capacity(h, C.byref(cap)))
        self.max_obstacles = int(cap.value)
        """the obstacle capacity O per planner: max(max_obstacles, the largest obstacle count of the planners at open)"""
        self._tasks = False                            # a set_goals / set_obstacles call was issued
        u, st, act = C.c_void_p(), C.c_void_p(), C.c_void_p()
        check(lib.b200mppi_loop_controls(h, C.byref(u), C.byref(st)))
        check(lib.b200mppi_loop_active(h, C.byref(act)))
        self.stream = int(st.value or 0)

        def unreadable(out):
            raise _lib.B200MPPIError("a device loop's arrays are read through __cuda_array_interface__ (e.g. "
                                     "torch.as_tensor(a, device='cuda'))")
        self._u = DeviceArray(self, (self.K, self.T, 2), np.float32, unreadable, dev_ptr=lambda: u.value,
                              stream=self.stream)
        self.active = DeviceArray(self, (self.K,), np.int32, unreadable, dev_ptr=lambda: act.value, stream=self.stream)
        """(K,) int32 running flags on the device, in ``batch.planners`` order"""
        self.solves = self.shifts = self.status = None
        batch._loop = self
        for i, p in enumerate(batch.planners):
            for obj in (p, getattr(p, "lin_tdm", None), getattr(p, "ang_tdm", None)):
                if obj is not None:
                    obj._device_loop = batch.order[i]

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()
        return False

    def __del__(self):
        if getattr(self, "_handle", None) is not None:
            try:
                self.close()
            except Exception:
                pass

    def _live(self, fn):
        if self._handle is None:
            raise ValueError("DeviceLoop.%s: the loop is closed" % fn)
        self._refuse_foreign_capture(fn)

    def _refuse_foreign_capture(self, fn):
        """ValueError while torch (if imported) captures a CUDA graph on a stream other than the loop's."""
        torch = sys.modules.get("torch")
        if torch is None or not torch.cuda.is_initialized() or not torch.cuda.is_current_stream_capturing():
            return
        cur = int(torch.cuda.current_stream().cuda_stream)
        if cur != self.stream:
            raise ValueError("DeviceLoop.%s: torch is capturing a CUDA graph on stream 0x%x, the loop runs on 0x%x "
                             "(batch.set_stream() to the capturing stream before the loop opens)" % (fn, cur, self.stream))

    def _array(self, obj, fn, what, shape, typestrs, strided_rows=False):
        """Pointer, typestr and row stride of ``obj``'s __cuda_array_interface__ (v3) after checking its shape, dtype,
        strides and device; if it names a stream, the batch's stream waits for that stream's work (an event)."""
        name = "DeviceLoop.%s" % fn
        try:
            cai = obj.__cuda_array_interface__
        except AttributeError:
            raise TypeError("%s: %s has no __cuda_array_interface__ (a torch or CuPy array, or a DeviceArray, in GPU "
                            "memory)" % (name, what))
        shape_o, typestr = tuple(int(v) for v in cai["shape"]), cai["typestr"]
        if shape_o != shape:
            raise ValueError("%s: %s of shape %s, expected %s" % (name, what, shape_o, shape))
        if typestr not in typestrs:
            raise ValueError("%s: %s of dtype %s, expected one of %s" % (name, what, typestr, ", ".join(typestrs)))
        item = int(typestr[2:])
        dense = tuple(int(np.prod(shape[d + 1:])) * item for d in range(len(shape)))
        strides = cai.get("strides")
        strides = dense if strides is None else tuple(int(v) for v in strides)
        row = strides[0] if len(shape) > 1 else item
        ok = strides[1:] == dense[1:] and (shape[0] == 1 or (row >= dense[0] if strided_rows else row == dense[0]))
        if not ok:
            raise ValueError("%s: %s with strides %s (%s)" % (name, what, strides, "rows may be strided, their elements "
                             "must be contiguous" if strided_rows else "must be C-contiguous"))
        if shape[0] == 1:
            row = dense[0]
        dev = getattr(obj, "device", None)
        if dev is not None:
            dtype_, index = getattr(dev, "type", "cuda"), getattr(dev, "index", getattr(dev, "id", None))
            if dtype_ != "cuda" or (index is not None and int(index) != self.device):
                raise ValueError("%s: %s is on device %s, the batch on cuda:%d" % (name, what, dev, self.device))
        stream = cai.get("stream")
        if stream is not None:
            check(lib.b200mppi_loop_wait_stream(self._handle, C.c_void_p(int(stream))))
        return C.c_void_p(int(cai["data"][0])), typestr, row

    def solve(self, out=None):
        """One solve of every running planner.  Returns a DeviceArray, a (K, T, 2) float32 view of the loop's own buffer
        (its __cuda_array_interface__ names the batch's stream) that the next solve() overwrites; with ``out``, a
        caller's (K, T, 2) float32 C-contiguous device array, the controls go there and ``out`` is returned.  Row k is
        planner k's new controls, NaN once it has stopped."""
        self._live("solve")
        if out is None:
            check(lib.b200mppi_loop_solve(self._handle, C.c_void_p(self._u._dev_ptr())))
            return self._u
        p, _, _ = self._array(out, "solve", "out", (self.K, self.T, 2), ("<f4",))
        check(lib.b200mppi_loop_solve(self._handle, p))
        return out

    def shift_and_update(self, x):
        """Every running planner takes its new pose x[k] ((K, 3) float64 or float32 on the batch's device; rows may be
        strided, their elements not): its controls shift by one row and its next solve plans from float32(x[k])."""
        self._live("shift_and_update")
        p, typestr, row = self._array(x, "shift_and_update", "x", (self.K, 3), ("<f8", "<f4"), strided_rows=True)
        check(lib.b200mppi_loop_shift_and_update(self._handle, p, _lib.POSE_F64 if typestr == "<f8" else _lib.POSE_F32,
                                                 row))

    def stop(self, done):
        """Planner k stops for good where done[k] ((K,) int32, bool or uint8 on the device) is nonzero."""
        self._live("stop")
        p, typestr, _ = self._array(done, "stop", "done", (self.K,), ("<i4", "|b1", "|u1"))
        check(lib.b200mppi_loop_stop(self._handle, p, 4 if typestr == "<i4" else 1))

    def set_goals(self, g):
        """Every running planner's later solves plan toward float32(g[k]) ((K, 2) float64 or float32 on the batch's
        device; rows may be strided, their elements not), as ``p.params['xgoal'] = g[k]`` before them.  Not checked:
        NaN and inf pass, as the host passes them."""
        self._live("set_goals")
        p, typestr, row = self._array(g, "set_goals", "g", (self.K, 2), ("<f8", "<f4"), strided_rows=True)
        self._tasks = True
        check(lib.b200mppi_loop_set_goals(self._handle, p, _lib.POSE_F64 if typestr == "<f8" else _lib.POSE_F32, row))

    def set_obstacles(self, obs, counts=None):
        """Barebone loops: every running planner's later solves avoid the first counts[k] obstacles [x, y, r] of
        obs[k] ((K, O', 3) float64 or float32 on the device, O' <= ``max_obstacles``; planner rows may be strided, the
        triples of a planner C-contiguous; counts (K,) int32 on the device, default O'), as
        ``p.params['obstacle_positions'] = obs[k, :n, :2]`` and ``p.params['obstacle_radius'] = obs[k, :n, 2]``
        before them.  A count outside [0, O'] stops that planner for good with status "bad_obstacles"."""
        self._live("set_obstacles")
        name = "DeviceLoop.set_obstacles"
        if self.batch.kind != "barebone":
            raise ValueError("%s: a %s loop (only barebone planners take obstacles)" % (name, self.batch.kind))
        try:
            shape = tuple(int(v) for v in obs.__cuda_array_interface__["shape"])
        except AttributeError:
            shape = None                               # refused by _array
        if shape is not None and (len(shape) != 3 or shape[0] != self.K or shape[2] != 3):
            raise ValueError("%s: obs of shape %s, expected (%d, O', 3)" % (name, shape, self.K))
        O = shape[1] if shape is not None else 0
        if O > self.max_obstacles:
            raise ValueError("%s: %d obstacles per planner, the loop's capacity is %d (device_loop(max_obstacles=...))"
                             % (name, O, self.max_obstacles))
        p, typestr, row = self._array(obs, "set_obstacles", "obs", (self.K, O, 3), ("<f8", "<f4"), strided_rows=True)
        c = None
        if counts is not None:
            c, _, _ = self._array(counts, "set_obstacles", "counts", (self.K,), ("<i4",))
        self._tasks = True
        check(lib.b200mppi_loop_set_obstacles(self._handle, p, _lib.POSE_F64 if typestr == "<f8" else _lib.POSE_F32, O,
                                              row, c))

    def close(self):
        """Wait for the stream, commit every planner (as after the host loop) and free the loop.  Idempotent.  Raises,
        with the loop left open, while the batch's stream captures a CUDA graph."""
        h = getattr(self, "_handle", None)
        if h is None:
            return
        self._refuse_foreign_capture("close")
        b = self.batch
        S = (_lib.LoopSummary * self.K)()
        tasks, obs = None, None
        if self._tasks:                                # the task updates' commit: close_ex
            tasks = (_lib.LoopTask * self.K)()
            obs = np.zeros((self.K, self.max_obstacles, 3), np.float64)
            rc = lib.b200mppi_loop_close_ex(h, S, tasks, ptr(obs) if self.max_obstacles else None)
        else:
            rc = lib.b200mppi_loop_close(h, S)
        if rc == _lib.EINVAL:                          # refused before any work: the loop stays open
            check(rc)
        self._handle = None
        try:
            check(rc)
        finally:
            b._loop = None
            for p in b.planners:
                for obj in (p, getattr(p, "lin_tdm", None), getattr(p, "ang_tdm", None)):
                    if obj is not None:
                        obj._device_loop = None
        solves, shifts, status = np.zeros(self.K, np.int64), np.zeros(self.K, np.int64), [None] * self.K
        for j, p in enumerate(b.planners):
            s, i = S[j], b.order[j]
            solves[i], shifts[i], status[i] = s.solves, s.shifts, LOOP_STATUS[s.status]
            if s.solves > 0 and not b._tdm[j]:
                p.u_prev_d = p._u_prev_buf             # as each planner's own solve() does (mppi.py:292,362)
            if s.shifts > 0:
                p.params["x0"] = np.array(s.x[:], dtype=np.float64)     # shift_and_update(x[k], ...)
            if tasks is not None and tasks[j].took_goal:
                p.params["xgoal"] = np.array(tasks[j].goal[:], dtype=np.float64)
            if tasks is not None and tasks[j].took_obstacles:
                n = int(tasks[j].num_obstacles)
                p.params["obstacle_positions"] = obs[j, :n, :2].copy()
                p.params["obstacle_radius"] = obs[j, :n, 2].copy()
        self.solves, self.shifts, self.status = solves, shifts, status
