"""N > 1 path on CPU: two gloo ranks shard the control sequences, each forms its softmax partial
(beta_r, S_r, V_r[2T]) exactly as the engine's update_partial/update_rank kernels define it, the
partials are all-gathered with torch.distributed and merged by the library's host combine
(b200mppi_combine_partials_host, the same math as update_apply_kernel).  Every rank must end with the
u_seq the oracle computes in a single process."""
import os
import socket

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

N, T, WS = 300, 11, 2


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    return port


def _inputs():
    rng = np.random.default_rng(21)
    costs = rng.uniform(700, 712, N).astype(np.float32)
    noise = (rng.standard_normal((N, T, 2)) * [2, 3]).astype(np.float32)
    u0 = np.stack([rng.uniform(0, 2, T), rng.uniform(-1, 1, T)], 1).astype(np.float32)
    return costs, noise, u0


def _rank_main(rank, port, out_dir):
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=WS)
    import __graft_entry__
    __graft_entry__.build_engine()
    from mppi_numba_b200 import _lib
    costs, noise, u0 = _inputs()
    lam = np.float32(1.0)
    n0, n1 = N * rank // WS, N * (rank + 1) // WS            # the library's sharding rule (b200mppi.h)
    c, e = costs[n0:n1], noise[n0:n1]
    beta = c.min()
    w = np.exp((-1.0 / float(lam)) * (c - beta).astype(np.float64)).astype(np.float32)
    V = np.einsum("n,ntk->tk", w.astype(np.float64), e.astype(np.float64)).astype(np.float32)
    part = torch.from_numpy(np.concatenate([[beta, w.sum(dtype=np.float64)], V.ravel()]).astype(np.float32))
    gathered = torch.empty((WS * (2 * T + 2),), dtype=torch.float32)          # flat: gloo wants 1-D
    dist.all_gather_into_tensor(gathered, part)
    g = np.ascontiguousarray(gathered.numpy().reshape(WS, 2 * T + 2))
    out = np.empty((T, 2), dtype=np.float32)
    vr, wr = np.array([0, 3], np.float32), np.array([-np.pi, np.pi], np.float32)
    _lib.check(_lib.lib.b200mppi_combine_partials_host(_lib.ptr(g), WS, T, lam, _lib.ptr(u0), _lib.ptr(vr),
                                                       _lib.ptr(wr), _lib.ptr(out)))
    np.save(os.path.join(out_dir, "u_rank%d.npy" % rank), out)
    dist.barrier()
    dist.destroy_process_group()


def test_two_rank_exchange_matches_single_process_oracle(tmp_path):
    from oracle import mppi_ref as MR
    port = _free_port()
    mp.spawn(_rank_main, args=(port, str(tmp_path)), nprocs=WS, join=True)
    costs, noise, u0 = _inputs()
    want, _ = MR.update_useq(1.0, costs, noise, [0, 3], [-np.pi, np.pi], u0)
    us = [np.load(os.path.join(str(tmp_path), "u_rank%d.npy" % r)) for r in range(WS)]
    assert (us[0] == us[1]).all()                      # every rank holds the identical update
    np.testing.assert_allclose(us[0], want, rtol=1e-5, atol=2e-6)


def test_generator_shards_are_slices_of_the_global_stream():
    """Rank r's noise generators are the global generators n*T+t of its rollouts (b200mppi.h:
    results do not depend on world_size)."""
    from oracle import xoroshiro as X
    full = X.create_states(N * T, 3)
    for ws in (2, 3):
        for r in range(ws):
            n0, n1 = N * r // ws, N * (r + 1) // ws
            z = X.splitmix64(3)
            s = (z, z)
            for _ in range(n0 * T):
                s = X.jump_scalar(*s)
            assert (int(full[n0 * T, 0]), int(full[n0 * T, 1])) == s
            assert n1 > n0


# ------------------------------------------------------------------------------------------------
# Set-up of the peer-memory exchange (MPPI_Numba._connect_peers): every rank exports an IPC handle, the handles
# are all-gathered, every rank imports them, and ALL ranks must agree on the outcome (one rank failing sends
# every rank to the collective-library exchange).  Run on two gloo ranks against tests/fake_backend.py.
def _peer_main(rank, port, out_dir):
    import contextlib
    import json
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=WS)
    import __graft_entry__
    __graft_entry__.build_engine()
    import mppi_numba_b200 as E
    import mppi_numba_b200.mppi as M
    import mppi_numba_b200.terrain as Tm
    from tests.fake_backend import FakeLib, disarm
    torch.cuda.device = lambda idx: contextlib.nullcontext()        # no CUDA in this process

    class Lib(FakeLib):
        fail_export = False

        def b200mppi_planner_p2p_export(self, h, out, n):
            self.calls.append(("planner_p2p_export", (n,)))
            if self.fail_export:
                return -3
            for i in range(64):
                out[i] = (rank * 64 + i) & 0xFF
            return 0

        def b200mppi_planner_p2p_import(self, h, handles, n):
            self.uploads["p2p_import"] = bytes(bytearray(handles[i] for i in range(n)))
            self.calls.append(("planner_p2p_import", (n,)))
            return 0

        def b200mppi_last_error(self):
            return b"no peer access"
    fake = Lib()
    M.lib = Tm.lib = fake
    cfg = E.Config(T=1.0, dt=0.1, num_grid_samples=4, num_control_rollouts=128, max_map_dim=(20, 20),
                   max_speed_padding=1.0, use_tdm=True)
    res = {}
    try:
        pl = E.MPPI_Numba(cfg, rank=rank, world_size=WS)
        created = [c for c in fake.calls if c[0] == "planner_create"][0][1]
        res["create"] = [created["rank"], created["world_size"], pl.shard_maps, pl.m_local, pl.n_local, pl.n_reduce]
        # 1. everybody succeeds
        os.environ.pop("B200MPPI_EXCHANGE", None)
        res["ok"] = bool(pl._connect_peers())
        blob = fake.uploads["p2p_import"]
        res["handles_in_rank_order"] = [blob[0], blob[64]] == [0, 64] and len(blob) == 128
        # 2. rank 1 cannot export: every rank must fall back
        fake.fail_export = (rank == 1)
        fake.uploads.pop("p2p_import", None)
        res["one_fails"] = bool(pl._connect_peers())
        res["import_skipped"] = "p2p_import" not in fake.uploads
        # 3. the same with the exchange forced: an error on every rank
        os.environ["B200MPPI_EXCHANGE"] = "p2p"
        try:
            pl._connect_peers()
            res["forced"] = "no error"
        except RuntimeError as e:
            res["forced"] = str(e)
        # 4. B200MPPI_EXCHANGE=nccl: no handshake at all
        os.environ["B200MPPI_EXCHANGE"] = "nccl"
        n_before = len(fake.calls)
        res["nccl"] = bool(pl._connect_peers())
        res["nccl_calls"] = len(fake.calls) - n_before
    finally:
        disarm(fake)
    with open(os.path.join(out_dir, "peer_rank%d.json" % rank), "w") as f:
        json.dump(res, f)
    dist.barrier()
    dist.destroy_process_group()


def test_peer_exchange_setup_is_agreed_by_all_ranks(tmp_path):
    import json
    port = _free_port()
    mp.spawn(_peer_main, args=(port, str(tmp_path)), nprocs=WS, join=True)
    r = [json.load(open(os.path.join(str(tmp_path), "peer_rank%d.json" % k))) for k in range(WS)]
    for k in range(WS):
        assert r[k]["create"] == [k, WS, True, 2, 128, 64]        # maps sharded: M/ws maps, all N rollouts, N/ws reduced
        assert r[k]["ok"] is True and r[k]["handles_in_rank_order"]
        assert r[k]["one_fails"] is False and r[k]["import_skipped"]
        assert "rank 1: no peer access" in r[k]["forced"]
        assert r[k]["nccl"] is False and r[k]["nccl_calls"] == 0
