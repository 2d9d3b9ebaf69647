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
# the unknown-scale stage in forced chunks of 2048 end points at n = 300 on a lattice (tie groups split across chunks)
lat = np.stack(np.meshgrid(*[np.arange(7.0)] * 3, indexing="ij"), -1).reshape(-1, 3)[:300]
ctx.set_scale_chunk(2048)
g = ctx.solve(lat, lat * 2.0, capi.default_params(noise_bound=0.01, estimate_scaling=1))
print("scale chunks", ctx.last_scale_chunks(), g["scale"])
ctx.set_scale_chunk(0)
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
# ragged batch padded into one size class (debug flag 16777216): n = 1 ... 700 share one padded device batch
rg = [synth.make_problem(n, 0.5, 40 + n, "ball") for n in (700, 1, 2, 129, 33, 300)]
for rflags, est in ((16777216, 0), (16777216 | 2, 0), (16777216, 1)):
    ctx.set_flags(rflags)
    sols, cl = ctx.solve_batch([q["src"] for q in rg], [q["dst"] for q in rg],
                               capi.default_params(noise_bound=rg[0]["noise_bound"], estimate_scaling=est))
    print("ragged flags", rflags, "scale", est, [int(c) for c in sols["clique_size"]])
ctx.set_flags(0)
# the default graph kernel's long strips (forced through debug flag bits 28-31; the automatic choice needs batches of
# thousands): 5, 6 and 8 blocks refill every slot of the column ring, 8 fills one a third time.  A uniform batch at
# n = 1100 (9 row blocks), under the production, verifying, two-slope and 64-entry-queue instances, then the ragged class
# above, whose problems end inside and before whole strips
lg = [synth.config_problem("C2", 70 + b, n=1100) for b in range(3)]
ls, ld = np.ascontiguousarray(np.stack([q["src"] for q in lg])), np.ascontiguousarray(np.stack([q["dst"] for q in lg]))
for L in (5, 6, 8):
    for sflags in (0, 2 | 4, 134217728, 16384 | 4):
        ctx.set_flags(sflags | capi.strip_flags(L))
        sols, cl = ctx.solve_batch_array(ls, ld, capi.default_params(**dict(kw, noise_bound=lg[0]["noise_bound"])))
        print("strips", L, "flags", sflags, ctx.last_strip_blocks(), [int(s) for s in sols["n_edges"]])
    for rflags in (16777216, 16777216 | 134217728 | 16384):
        ctx.set_flags(rflags | capi.strip_flags(L))
        sols, cl = ctx.solve_batch([q["src"] for q in rg], [q["dst"] for q in rg],
                                   capi.default_params(noise_bound=rg[0]["noise_bound"], estimate_scaling=0))
        print("ragged strips", L, "flags", rflags, ctx.last_strip_blocks(), [int(c) for c in sols["clique_size"]])
ctx.set_flags(0)
if "--no-cert" not in sys.argv:  # solve then certify its retained results: the gather kernel on CHAIN and COMPLETE TIMs
    for tim in (0, 1):
        sc = [synth.make_problem(n, 0.5, 60 + n, "ball") for n in (40, 30, 36)]
        ctx.solve_batch([q["src"] for q in sc], [q["dst"] for q in sc],
                        capi.default_params(noise_bound=sc[0]["noise_bound"], estimate_scaling=1, rotation_tim_graph=tim))
        rc = ctx.certify_last(noise_bound=2 * sc[0]["noise_bound"], max_iterations=3)
        print("certify_last tim", tim, [(r["status"], len(r["suboptimality_traj"])) for r in rc])
# point-to-point ICP: both nearest-neighbour routes (brute force, and the grid with a far point forcing a fallback)
ic_src = rng.uniform(0, 0.3, size=(300, 3)).astype(np.float32)
ic_dst = (ic_src + rng.normal(scale=0.005, size=ic_src.shape)).astype(np.float32)
ic_dst[0] = np.nan
for iflags in (33554432, 67108864):
    ctx.set_flags(iflags)
    res, corr = ctx.icp_batch([ic_src, ic_src[:3]], [ic_dst, np.concatenate([ic_dst, [[1e9, 0, 0]]]).astype(np.float32)],
                              0.05, max_iteration=3)
    print("icp flags", iflags, [int(r) for r in res["n_correspondences"]], [int(r) for r in res["iterations"]])
ctx.set_flags(0)
# normals alone and point-to-plane ICP: a ragged batch with NaN normals, a non-finite point and an overflowing cloud
nm = [ic_src, ic_dst, np.zeros((4100, 3), dtype=np.float32), ic_src[:2]]
try:
    ctx.estimate_normals_batch(nm, 0.05)
except capi.TzrError as e:
    print("normals status", e.status.tolist())
    nrm = e.result
nrm[0][::4] = np.nan
for iflags in (33554432, 67108864):
    ctx.set_flags(iflags)
    res, corr = ctx.icp_point_to_plane_batch([ic_dst, ic_src[:3], ic_src], [ic_src, ic_dst, ic_src[:2]],
                                             [nrm[0], nrm[1], nrm[3]], 0.05, max_iteration=3)
    print("icp plane flags", iflags, [int(r) for r in res["n_correspondences"]], [int(r) for r in res["iterations"]])
    # generalized ICP: the same batch with source normals too (NaN rows on both sides)
    res, corr = ctx.icp_generalized_batch([ic_dst, ic_src[:3], ic_src], [ic_src, ic_dst, ic_src[:2]],
                                          [nrm[1], nrm[0][:3], nrm[0]], [nrm[0], nrm[1], nrm[3]], 0.05,
                                          max_iteration=3)
    print("icp generalized flags", iflags, [int(r) for r in res["n_correspondences"]],
          [int(r) for r in res["iterations"]])
ctx.set_flags(0)
# the chained entry with generalized ICP: both clouds' normals from its own FPFH stage
gp = ctx.register_cloud_pairs_icp([ic_src[1:], ic_dst[1:]], [(0, 1), (1, 0)],
                                  capi.default_params(noise_bound=0.01, estimate_scaling=0), 0.05,
                                  normal_search_radius=0.05, fpfh_search_radius=0.1, method="generalized",
                                  max_iteration=3)
print("register_cloud_pairs_icp generalized", gp[1].tolist(), [int(r) for r in gp[6]["iterations"]])
# robust kernels: both batch entries with a NaN normal, L1 at a zero residual (a problem onto itself) and Tukey with
# every residual beyond k, then the chained entry with each method
for kern in (("l1", 0.0), ("tukey", 1e-12), ("cauchy", 0.02)):
    res, _ = ctx.icp_point_to_plane_batch([ic_dst, ic_src, ic_src], [ic_src, ic_src, ic_dst[:2]],
                                          [nrm[0], nrm[0], nrm[1][:2]], 0.05, max_iteration=3, kernel=kern)
    print("icp plane robust", kern, [int(r) for r in res["n_correspondences"]], [int(r) for r in res["iterations"]])
    res, _ = ctx.icp_generalized_batch([ic_dst, ic_src, ic_src], [ic_src, ic_src, ic_dst[:2]],
                                       [nrm[1], nrm[0], nrm[0]], [nrm[0], nrm[0], nrm[1][:2]], 0.05, max_iteration=3,
                                       kernel=kern)
    print("icp generalized robust", kern, [int(r) for r in res["n_correspondences"]],
          [int(r) for r in res["iterations"]])
for method in ("point_to_plane", "generalized"):
    gp = ctx.register_cloud_pairs_icp([ic_src[1:], ic_dst[1:]], [(0, 1), (1, 0)],
                                      capi.default_params(noise_bound=0.01, estimate_scaling=0), 0.05,
                                      normal_search_radius=0.05, fpfh_search_radius=0.1, method=method,
                                      max_iteration=3, kernel=("tukey", 0.05))
    print("register_cloud_pairs_icp robust", method, gp[1].tolist(), [int(r) for r in gp[6]["iterations"]])
# voxel downsampling: a ragged batch with a NaN row, an all-NaN cloud and a cloud too wide for the voxel (INT_MAX check)
vx = [rng.uniform(0, 1, size=(500, 3)).astype(np.float32), np.full((3, 3), np.nan, dtype=np.float32),
      np.array([[0, 0, 0], [1e9, 0, 0]], dtype=np.float32), rng.uniform(0, 1, size=(1, 3)).astype(np.float32)]
vx[0][7] = np.nan
try:
    ctx.voxel_downsample_batch(vx, 0.1, return_trace=True)
except capi.TzrError as e:
    print("voxel status", e.status.tolist(), [len(o) for o in e.result[0]])
sols, cl = capi.solve_batch_multi([p["src"] for p in prs[:5]], [p["dst"] for p in prs[:5]],
                                  capi.default_params(**dict(kw, noise_bound=prs[0]["noise_bound"])))
print("multi", int(sols["valid"].sum()), "/ 5")
# the batched line process: two fragment-shaped graphs on the batched route (the Cholesky's shared-memory tiles) and
# one refused graph
sys.path.insert(0, os.path.join(ROOT, "tests"))
from line_process_fragments import fragment  # noqa: E402
lpg = []
for seed, K in ((1, 40), (2, 75)):
    gt_, e_, T_, L_, u_ = fragment(seed, K, n_wrong=1)
    lpg.append(dict(K=K, edges=e_, transforms=T_, information=L_, uncertain=u_))
lpg.append(dict(lpg[0], K=41))
lpr = ctx.global_optimization_batch(lpg, 0.05)
print("line process batch", [r["status"] for r in lpr], [r["trials"] for r in lpr])
# the batched GNC-TLS pose graph on the same graphs (one refused)
pgr = ctx.optimize_pose_graph_batch(lpg, 0.05)
print("pose graph batch", [r["status"] for r in pgr], [r["inner_iterations"] for r in pgr])
# many scan sequences in one multiway call with fused maps: two small sequences and one refused (an unsolvable pair)
mw_seqs = [[ic_src, ic_dst, ic_src[1:]], [ic_dst, ic_src], [ic_src, ic_dst[:2]]]
for opt in ("gnc_tls", "line_process"):
    mwr = ctx.register_multiway_batch(mw_seqs, [[(0, 1), (1, 2)], [(0, 1)], [(0, 1)]],
                                      capi.default_params(noise_bound=0.01, estimate_scaling=0), 0.05,
                                      normal_search_radius=0.05, fpfh_search_radius=0.1, max_iteration=3,
                                      optimizer=opt, map_voxel_size=0.05)
    print("multiway batch", opt, [r[7]["status"] for r in mwr], [len(r[7]["map"]) for r in mwr])
# the batched routes' Cholesky on given matrices: mixed sizes (panel stride 70), one that fails at column 40
dc_A = [np.eye(n) * 4.0 + np.tril(np.full((n, n), 0.01), -1) for n in (0, 5, 33, 70)]
dc_A[3][40, 40] = -1.0
_, _, dc_info = ctx.dense_cholesky_batch(dc_A, [np.ones(len(a)) for a in dc_A])
print("dense cholesky batch", dc_info.tolist())
ctx.close()
print("DONE")
