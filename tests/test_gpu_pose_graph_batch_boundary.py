"""Both batched pose-graph routes at their size edges (run on an H100: `pytest -m gpu`): the default cutoff (K = 128
batched, K = 129 through the single entry), the shared-memory cap (K = cap batched with TZR_LP_BATCH_MAX_K at the cap,
in the largest shared-memory configuration; K = cap + 1 clamped to the single entry with the variable at 1024), and
the line-process batch's failed-factorisation path beside another graph."""
import importlib

import numpy as np
import pytest

import dense_cholesky_reference as dc
import line_process_reference as lp
from line_process_fragments import fragment
from test_gpu_line_process import R_CORR as LP_CORR, check as lp_check
from test_gpu_line_process_batch import gd, restate as lp_restate, same_bytes as lp_same, single as lp_single
from test_gpu_pose_graph_batch import check as pg_check, restate as pg_restate, same_bytes as pg_same, \
    single as pg_single
from test_gpu_pose_graph import R_CORR as PG_CORR
from test_gpu_pose_graph_boundary import indefinite_graph

capi = importlib.import_module("teaser-plusplus_b200.capi")

pytestmark = pytest.mark.gpu

LP_DECISIONS = ("iterations", "trials", "stop_reason", "pruned")


@pytest.fixture(scope="module")
def ctx():
    c = capi.Context(0)
    yield c
    c.close()


def counted(ctx, fn):
    l0 = ctx.kernel_launches()
    out = fn()
    return out, ctx.kernel_launches() - l0


def gnc_batch_and_single(ctx, d):
    got, n_batch = counted(ctx, lambda: ctx.optimize_pose_graph_batch([d], PG_CORR)[0])
    want, n_single = counted(ctx, lambda: pg_single(ctx, d))
    assert got.pop("status") == 0
    return got, n_batch, want, n_single


def lp_batch_and_single(ctx, d):
    got, n_batch = counted(ctx, lambda: ctx.global_optimization_batch([d], LP_CORR)[0])
    want, n_single = counted(ctx, lambda: lp_single(ctx, d))
    assert got.pop("status") == 0
    return got, n_batch, want, n_single


def batched(ctx, K, seed):
    """Both optimisers on a K-node fragment that must take the batched route: 1 and 2 launches, the restatement's
    results, the single entry's decisions."""
    d = gd(fragment(seed, K, n_wrong=2))
    got, n, s, n_s = gnc_batch_and_single(ctx, d)
    assert n == 1 and n_s > 1
    pg_check(got, pg_restate(d))
    assert (got["iterations"], got["inner_iterations"]) == (s["iterations"], s["inner_iterations"])
    got, n, s, n_s = lp_batch_and_single(ctx, d)
    assert n == 2 and n_s > 2
    lp_check(got, lp_restate(d))
    for k in LP_DECISIONS:
        assert got[k] == s[k], k
    assert np.array_equal(got["kept"], s["kept"])


def single_route(ctx, K, seed):
    """Both optimisers on a K-node fragment that must take the single route: byte-identical to the single entry, with
    its launch count."""
    d = gd(fragment(seed, K, n_wrong=2))
    got, n, s, n_s = gnc_batch_and_single(ctx, d)
    assert n == n_s
    pg_same(got, s)
    pg_check(got, pg_restate(d))
    got, n, s, n_s = lp_batch_and_single(ctx, d)
    assert n == n_s
    lp_same(got, s)
    lp_check(got, lp_restate(d))


def test_default_cutoff(ctx, monkeypatch):
    monkeypatch.delenv("TZR_LP_BATCH_MAX_K", raising=False)
    batched(ctx, 128, 11)
    single_route(ctx, 129, 12)


def test_the_shared_memory_cap(ctx, monkeypatch):
    import torch
    optin = torch.cuda.get_device_properties(0).shared_memory_per_block_optin
    cap = dc.batch_cap(optin)
    assert dc.batch_smem(6 * cap) <= optin < dc.batch_smem(6 * (cap + 1))
    monkeypatch.setenv("TZR_LP_BATCH_MAX_K", str(cap))
    batched(ctx, cap, 13)  # the line process at n = 6 cap: the largest panel the device holds
    monkeypatch.setenv("TZR_LP_BATCH_MAX_K", "1024")
    single_route(ctx, cap + 1, 14)


def test_failed_factorisation_in_the_line_process_batch(ctx):
    """The indefinite graph's first H + lambda I does not factor (skip 2, a rejection), then the damping climbs until it
    does: the restatement's and the single entry's decisions, mu and kept set, alone and beside a fragment."""
    edges, T, L = indefinite_graph()
    d = dict(K=3, edges=edges, transforms=T, information=L, uncertain=None, initial_poses=None)
    tr = []
    want = lp.optimize(3, edges, T, L, LP_CORR, None, trace=tr)
    failed = [x for x in tr if "dnorm" not in x]  # a trial whose factorisation failed forms no step
    assert failed and tr[0] is failed[0]
    s = lp_single(ctx, d)
    for ds, at in (([d], 0), ([gd(fragment(9, 40, n_wrong=1)), d], 1), ([d, gd(fragment(9, 40, n_wrong=1))], 0)):
        got = ctx.global_optimization_batch(ds, LP_CORR)[at]
        assert got["status"] == 0
        lp_check(got, want)
        for k in LP_DECISIONS:
            assert got[k] == s[k] == want[k], k
        assert np.asarray(got["mu"]).tobytes() == np.asarray(s["mu"]).tobytes()
        assert np.array_equal(got["kept"], s["kept"]) and np.array_equal(got["kept"], want["kept"])
