"""Exercise every kernel once on small inputs (meant to run under compute-sanitizer)."""
import importlib
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
capi = importlib.import_module("teaser-plusplus_b200.capi")
synth = importlib.import_module("teaser-plusplus_b200.synth")

ctx = capi.Context(0)
pr = synth.config_problem("C2cube", 1, n=333)
kw = dict(noise_bound=pr["noise_bound"], estimate_scaling=0, rotation_cost_threshold=1e-12)
bits, deg, ne = ctx.graph_build(pr["src"], pr["dst"], 2 * pr["noise_bound"])
for mode in (0, 1, 2):
    c, proven = ctx.max_clique(bits, 333, mode=mode)
    print("clique mode", mode, len(c), proven)
for alg in (0, 1, 2):
    for graph in (0, 1):
        g = ctx.solve(pr["src"], pr["dst"], capi.default_params(rotation_estimation_algorithm=alg,
                                                                rotation_tim_graph=graph, **kw))
        print("solve alg", alg, "graph", graph, g["valid"], len(g["clique"]))
g = ctx.solve(pr["src"][:120], pr["dst"][:120] * 1.5, capi.default_params(noise_bound=pr["noise_bound"], estimate_scaling=1))
print("scale small", g["scale"])
q = synth.make_problem(1600, 0.5, 5, "ball")
g = ctx.solve(q["src"], q["dst"] * 2.0, capi.default_params(noise_bound=2 * q["noise_bound"], estimate_scaling=1))
print("scale large", g["scale"], len(g["clique"]))
g = ctx.solve(pr["src"], pr["dst"], capi.default_params(inlier_selection_mode=3, **kw))
print("none mode", len(g["clique"]))
prs = [synth.config_problem("C4", b, n=257) for b in range(70)]
src = np.ascontiguousarray(np.stack([p["src"] for p in prs]))
dst = np.ascontiguousarray(np.stack([p["dst"] for p in prs]))
sols, cl = ctx.solve_batch_array(src, dst, capi.default_params(**dict(kw, noise_bound=prs[0]["noise_bound"])))
print("batch", int(sols["valid"].sum()), "/ 70")
rng = np.random.default_rng(0)
A = np.triu(rng.uniform(size=(200, 200)) < 0.4, 1)
A = A | A.T
pad = np.zeros((200, 256), dtype=np.uint8)
pad[:, :200] = A
b2 = np.packbits(pad, axis=1, bitorder="little").view(np.uint64).reshape(200, 4)
c, proven = ctx.max_clique(b2, 200, mode=0)
print("random graph clique", len(c), proven)
t, m = ctx.tls_translation(pr["src"][:50], pr["src"][:50] + 1.0, 0.01)
e, i = ctx.scalar_tls([0.5, 1, 0.6, 0.7, 1.2], [0.9, 0.9, 0.4, 0.5, 0.4])
r = ctx.rotation_solve(1, pr["src"][:60], pr["src"][:60], 0.01)
print("stage calls ok", t, e)
# dense graph: first exact pass hits its 50 ms deadline (always, under the sanitizer), then clique_lp_kernel + second pass
rng2 = np.random.default_rng(5)
ds = rng2.uniform(0, 0.15, size=(500, 3))
dd = ds + (rng2.random((500, 3)) - 0.5) * 0.1
dd[:150] += 7.0
g = ctx.solve(ds, dd, capi.default_params(noise_bound=0.05, estimate_scaling=0, max_clique_time_limit=20.0))
print("dense", len(g["clique"]), int(g["sol"].clique_proven_optimal))
# upstream / downstream stages
mp = synth.matcher_problem(300, 260, 90, seed=3)
for cc in (False, True):
    for tt in (False, True):
        pairs = ctx.match_correspondences(mp["src_pts"], mp["dst_pts"], mp["src_feat"], mp["dst_feat"], False, cc, tt,
                                          0.95, tuple_seed=5)
        print("matcher crosscheck", cc, "tuple", tt, len(pairs))
idx, dist = ctx.feature_nn(mp["src_feat"], mp["dst_feat"])
bp, _ = synth.bunny_fpfh()
f, nrm = ctx.compute_fpfh(bp, 0.03, 0.05, return_normals=True)
print("fpfh", f.shape, float(f.sum()))
if "--no-cert" not in sys.argv:  # cuSOLVER's own kernels are slow under the sanitizer; ours are covered by the blocks
    N = 12
    v1 = rng.uniform(-1, 1, size=(3, N))
    Rr = synth.random_rotation(rng)
    v2 = Rr @ v1
    th = np.ones(N)
    th[-2:] = -1
    v2[:, -2:] += 3.0
    M0, mu = ctx.certifier_initial_matrix(Rr, v1, v2, th)
    Wd = ctx.certifier_dual_projection(M0, th)
    r = ctx.certify(Rr, v1, v2, th, max_iterations=3)
    print("certify", mu, len(r["suboptimality_traj"]))
# round 2: the tensor-core graph kernel (wgmma / TMA / mbarrier pipeline), the one-MUFU strip kernel, the re-check queue
for flags in (1024, 1024 | 2, 2048, 2048 | 2, 2048 | 1):
    ctx.set_flags(flags | 4)
    for cfg, n in (("C2", 300), ("C2cube", 200)):
        q = synth.config_problem(cfg, 3, n=n)
        b3, d3, e3 = ctx.graph_build(q["src"], q["dst"], 2 * q["noise_bound"])
        print("graph flags", flags, cfg, n, e3, ctx.debug_counters()["filter_mismatches"])
    sols, cl = ctx.solve_batch_array(src[:9], dst[:9], capi.default_params(**dict(kw, noise_bound=prs[0]["noise_bound"])))
    print("batch flags", flags, int(sols["valid"].sum()), "/ 9")
ctx.set_flags(0)
sols, cl = capi.solve_batch_multi([p["src"] for p in prs[:5]], [p["dst"] for p in prs[:5]],
                                  capi.default_params(**dict(kw, noise_bound=prs[0]["noise_bound"])))
print("multi", int(sols["valid"].sum()), "/ 5")
ctx.close()
print("DONE")
