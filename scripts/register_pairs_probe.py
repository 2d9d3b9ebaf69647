"""Registering many cloud pairs: the chain of existing batch calls, built by hand on the host, against
tzr_register_cloud_pairs, in the same run.

chain:    compute_fpfh_batch over the clouds -> match_correspondences_batch over the pairs -> float64 rows of the float
          points at the correspondences (host) -> solve_batch over the pairs
one call: register_cloud_pairs(clouds, pairs)

The clouds are the wavy surface scans of scripts/frontend_batch_probe.py (a moved copy sharing 2/3 of its points).
Two topologies: independent pairs (2P clouds, pair k = (2k, 2k + 1)) and a sequence (P + 1 clouds, every scan a moved
copy of the one before, pair k = (k, k + 1), so every inner cloud is in two pairs).  Matching uses the example's flags
(examples/teaser_cpp_fpfh: absolute scale off, cross check on, no tuple test).  Both paths must give identical
correspondences, records (except stage_ms) and cliques; each time is the median of --reps calls after a warm-up call.

usage: python scripts/register_pairs_probe.py [--reps 3] [--sizes 1000,5000] [--pairs 16,256] [--out rows.json]
Prints the card's name and power limit, then one JSON line per (n, P, topology)."""
import argparse
import importlib
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))
capi = importlib.import_module("teaser-plusplus_b200.capi")
fbp = importlib.import_module("frontend_batch_probe")

FLAGS = (False, True, False, 0.0)
STAGE_OFF = capi.SOLUTION_DTYPE.fields["stage_ms"][1]


def clouds_of(n, P, topology, seed):
    if topology == "independent":
        clouds = []
        for k in range(P):
            clouds += list(fbp.make_pair(n, seed + k))
        return clouds, [(2 * k, 2 * k + 1) for k in range(P)]
    clouds = [fbp.make_pair(n, seed)[0]]
    for k in range(P):  # scan k + 1: scan k moved, 2/3 of its points kept (make_pair's rule, applied to scan k)
        rng = np.random.default_rng(seed + 1 + k)
        src = clouds[-1].astype(np.float64)
        keep = n - n // 3
        dst = np.concatenate([src[:keep], fbp.surface(rng, n - keep)])[rng.permutation(n)]
        a = rng.normal(size=3)
        a *= 0.05 / np.linalg.norm(a)
        K = np.array([[0, -a[2], a[1]], [a[2], 0, -a[0]], [-a[1], a[0], 0]])
        R = np.eye(3) + np.sin(0.05) * K / 0.05 + (1 - np.cos(0.05)) * (K @ K) / 0.05 ** 2
        clouds.append((dst @ R.T + np.array([0.05, 0.0, 0.0])).astype(np.float32))
    return clouds, [(k, k + 1) for k in range(P)]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--sizes", default="1000,5000")
    ap.add_argument("--pairs", default="16,256")
    ap.add_argument("--out", default=None, help="JSON file for the rows (default: stdout only)")
    a = ap.parse_args()
    ctx = capi.Context(0)
    name, power = fbp.card()
    print(json.dumps(dict(card=name, power_limit=power)), flush=True)
    prm = capi.default_params(noise_bound=0.01, estimate_scaling=0)
    rows = []
    for n in [int(x) for x in a.sizes.split(",")]:
        rn, rf = fbp.RADII[n]
        for P in [int(x) for x in a.pairs.split(",")]:
            for topology in ("independent", "sequence"):
                clouds, pairs = clouds_of(n, P, topology, 1000 * n + P)
                seeds = list(range(P))

                def chain():
                    feats = ctx.compute_fpfh_batch(clouds, rn, rf)
                    corr = ctx.match_correspondences_batch([clouds[s] for s, _ in pairs], [clouds[d] for _, d in pairs],
                                                           [feats[s] for s, _ in pairs], [feats[d] for _, d in pairs],
                                                           *FLAGS, tuple_seeds=seeds)
                    src = [np.ascontiguousarray(clouds[s][c[:, 0]], dtype=np.float64) for (s, _), c in zip(pairs, corr)]
                    dst = [np.ascontiguousarray(clouds[d][c[:, 1]], dtype=np.float64) for (_, d), c in zip(pairs, corr)]
                    sols, cliques = ctx.solve_batch(src, dst, prm)
                    return corr, sols, cliques

                def one_call():
                    sols, status, index, corr, cliques, _ = ctx.register_cloud_pairs(clouds, pairs, prm, rn, rf, *FLAGS,
                                                                                     tuple_seeds=seeds)
                    assert (status == 0).all()
                    return corr, sols, cliques

                t_chain = fbp.timed(chain, a.reps)
                t_one = fbp.timed(one_call, a.reps)
                (c0, s0, q0), (c1, s1, q1) = t_chain[3], t_one[3]
                same = all(np.array_equal(x, y) for x, y in zip(c0, c1)) and \
                    all(s0[k:k + 1].tobytes()[:STAGE_OFF] == s1[k:k + 1].tobytes()[:STAGE_OFF] for k in range(P)) and \
                    all(np.array_equal(x, y) for x, y in zip(q0, q1))
                row = dict(n=n, P=P, topology=topology, clouds=len(clouds), reps=a.reps,
                           chain_ms=1e3 * t_chain[0], chain_ms_range=[1e3 * t_chain[1], 1e3 * t_chain[2]],
                           one_call_ms=1e3 * t_one[0], one_call_ms_range=[1e3 * t_one[1], 1e3 * t_one[2]],
                           speedup=t_chain[0] / t_one[0], mean_corr=float(np.mean([len(c) for c in c1])),
                           identical=bool(same), card=name, power_limit=power)
                rows.append(row)
                print(json.dumps(row), flush=True)
                assert same, f"chain and one call differ at n={n} P={P} {topology}"
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as fh:
            json.dump(rows, fh, indent=1)
    ctx.close()


if __name__ == "__main__":
    main()
