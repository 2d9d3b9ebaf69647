// TEST INFRASTRUCTURE ONLY — CPU restatement of teaser::Matcher::calculateCorrespondences
// (reference: teaser/src/matcher.cc:21-337).  Nothing outside tests/, __graft_entry__.smoke() and bench.py's CPU
// legs may link or call this file; the product path (libteaser_b200.so) never does.
//
// PARITY STATUS: **unpinned**.  The reference's two matcher tests (test/teaser/matcher-test.cc:17-78) feed FPFH
// descriptors computed by PCL, and the nearest-neighbour search is FLANN's KDTreeSingleIndex (flann 1.9.x, a system
// package the reference finds with find_package; neither PCL nor FLANN is part of the reference tree).
// What is restated here:
//   * normalizePoints (matcher.cc:55-113): float arithmetic, sequential accumulation in index order;
//   * advancedMatching (matcher.cc:114-297): larger cloud becomes "i"; NN of every j in the i-features; the reverse
//     NN only for i that were hit (`i_to_j`, :155-164); corres = corres_ij ++ corres_ji; optional cross check
//     (:180-215, mutual nearest neighbours, emitted in ascending i); optional tuple test (:223-281);
//     swap back, sort, unique (:283-297).
//   * the NN itself: KDTreeSingleIndex with eps = 0 is an exact search under flann::L2<float>, whose accumulation
//     order is groups of four, `result += d0*d0 + d1*d1 + d2*d2 + d3*d3`, then the tail one by one
//     (published FLANN dist.h, struct L2).  Distances are restated in exactly that float order; among equal
//     distances the LOWEST index wins here (FLANN's choice depends on its tree layout).
//   * the tuple test draws `rand() % ncorr` after `srand(time(NULL))` (matcher.cc:225-234): the reference output is
//     nondeterministic by construction.  Here the three draws of trial t are the top 31 bits of
//     splitmix64(seed + 3 t + k), k = 0..2 — same distribution, reproducible, and parallelisable.
#include <algorithm>
#include <cmath>
#include <cstdint>
#include <cstring>
#include <utility>
#include <vector>

namespace {

typedef int64_t i64;

inline uint64_t splitmix64(uint64_t x) {
  x += 0x9E3779B97F4A7C15ull;
  x = (x ^ (x >> 30)) * 0xBF58476D1CE4E5B9ull;
  x = (x ^ (x >> 27)) * 0x94D049BB133111EBull;
  return x ^ (x >> 31);
}

// flann::L2<float>::operator() accumulation order (no early exit: it only ever skips non-minimal candidates)
inline float l2_flann(const float* a, const float* b, int dim) {
  float result = 0.f;
  int k = 0;
  for (; k + 3 < dim; k += 4) {
    const float d0 = a[k] - b[k], d1 = a[k + 1] - b[k + 1], d2 = a[k + 2] - b[k + 2], d3 = a[k + 3] - b[k + 3];
    result += d0 * d0 + d1 * d1 + d2 * d2 + d3 * d3;
  }
  for (; k < dim; ++k) {
    const float d0 = a[k] - b[k];
    result += d0 * d0;
  }
  return result;
}

// exact 1-NN of q among db[0..n), lowest index among ties
int nn1(const float* q, const float* db, int n, int dim) {
  int best = 0;
  float bd = l2_flann(q, db, dim);
  for (int i = 1; i < n; ++i) {
    const float d = l2_flann(q, db + (size_t)i * dim, dim);
    if (d < bd || (bd != bd && d == d)) {  // a NaN distance never beats a number (it cannot in FLANN's heap either)
      bd = d;
      best = i;
    }
  }
  return best;
}

// matcher.cc:55-113.  pts are modified in place; returns global_scale_.
float normalize_points(std::vector<float>* cloud, bool use_absolute_scale) {
  float scale = 0.f;
  for (int c = 0; c < 2; ++c) {
    std::vector<float>& p = cloud[c];
    const int n = (int)(p.size() / 3);
    float mx = 0.f, my = 0.f, mz = 0.f;
    for (int i = 0; i < n; ++i) {  // mean = mean + p, sequential (:68-71)
      mx = mx + p[3 * i];
      my = my + p[3 * i + 1];
      mz = mz + p[3 * i + 2];
    }
    mx = mx / n;
    my = my / n;
    mz = mz / n;
    float max_scale = 0.f;
    for (int i = 0; i < n; ++i) {
      p[3 * i] -= mx;
      p[3 * i + 1] -= my;
      p[3 * i + 2] -= mz;
    }
    for (int i = 0; i < n; ++i) {
      const float x = p[3 * i], y = p[3 * i + 1], z = p[3 * i + 2];
      const float t = std::sqrt((x * x + y * y) + z * z);  // Vector3f::norm()
      if (t > max_scale) max_scale = t;
    }
    if (max_scale > scale) scale = max_scale;
  }
  const float g = use_absolute_scale ? 1.0f : scale;
  if (g != 1.0f)
    for (int c = 0; c < 2; ++c)
      for (float& v : cloud[c]) v /= g;
  return g;
}

inline float dist3(const float* a, const float* b) {
  const float x = a[0] - b[0], y = a[1] - b[1], z = a[2] - b[2];
  return std::sqrt((x * x + y * y) + z * z);
}

}  // namespace

extern "C" {

// Returns the number of correspondences written to pairs (int32 [first, second] rows, capacity rows), or -1 when
// capacity is too small.
i64 orc_match_correspondences(const float* src_pts, int ns, const float* dst_pts, int nd, const float* src_feat,
                              const float* dst_feat, int dim, int use_absolute_scale, int use_crosscheck,
                              int use_tuple_test, float tuple_scale, uint64_t tuple_seed, int32_t* pairs,
                              i64 capacity, float* global_scale_out) {
  std::vector<float> cloud[2];
  cloud[0].assign(src_pts, src_pts + (size_t)ns * 3);
  cloud[1].assign(dst_pts, dst_pts + (size_t)nd * 3);
  const float g = normalize_points(cloud, use_absolute_scale != 0);
  if (global_scale_out) *global_scale_out = g;
  const float* feat[2] = {src_feat, dst_feat};
  const int npts[2] = {ns, nd};

  int fi = 0, fj = 1;
  bool swapped = false;
  if (npts[fj] > npts[fi]) {  // :121-126
    std::swap(fi, fj);
    swapped = true;
  }
  const int nPti = npts[fi], nPtj = npts[fj];
  std::vector<int> i_to_j(nPti, -1), nn_of_j(nPtj);
#pragma omp parallel for schedule(static)
  for (int j = 0; j < nPtj; ++j) nn_of_j[j] = nn1(feat[fj] + (size_t)j * dim, feat[fi], nPti, dim);
  std::vector<uint8_t> hit(nPti, 0);
  for (int j = 0; j < nPtj; ++j) hit[nn_of_j[j]] = 1;
#pragma omp parallel for schedule(dynamic, 16)
  for (int i = 0; i < nPti; ++i)
    if (hit[i]) i_to_j[i] = nn1(feat[fi] + (size_t)i * dim, feat[fj], nPtj, dim);

  std::vector<std::pair<int, int>> corres;
  if (!use_crosscheck) {
    for (int i = 0; i < nPti; ++i)
      if (i_to_j[i] != -1) corres.emplace_back(i, i_to_j[i]);
    for (int j = 0; j < nPtj; ++j) corres.emplace_back(nn_of_j[j], j);
  } else {
    // Mi[i] = {i_to_j[i]} and Mj[j] = {nn_of_j[j]} hold one entry each, so the triple loop (:196-208) emits (i, j)
    // exactly when i_to_j[i] == j and nn_of_j[j] == i (mutual nearest neighbours), in ascending i.
    for (int i = 0; i < nPti; ++i) {
      const int j = i_to_j[i];
      if (j != -1 && nn_of_j[j] == i) corres.emplace_back(i, j);
    }
  }

  if (use_tuple_test && tuple_scale != 0.f) {  // :223-281
    const float scale = tuple_scale;
    const i64 ncorr = (i64)corres.size();
    const i64 trials = ncorr * 100;
    std::vector<uint8_t> keep((size_t)ncorr, 0);
    const float* pi = cloud[fi].data();
    const float* pj = cloud[fj].data();
    for (i64 t = 0; t < trials; ++t) {
      i64 r[3];
      for (int k = 0; k < 3; ++k) r[k] = (i64)(splitmix64(tuple_seed + 3ull * (uint64_t)t + k) >> 33) % ncorr;
      const float* a0 = pi + 3 * (size_t)corres[r[0]].first;
      const float* a1 = pi + 3 * (size_t)corres[r[1]].first;
      const float* a2 = pi + 3 * (size_t)corres[r[2]].first;
      const float* b0 = pj + 3 * (size_t)corres[r[0]].second;
      const float* b1 = pj + 3 * (size_t)corres[r[1]].second;
      const float* b2 = pj + 3 * (size_t)corres[r[2]].second;
      const float li0 = dist3(a0, a1), li1 = dist3(a1, a2), li2 = dist3(a2, a0);
      const float lj0 = dist3(b0, b1), lj1 = dist3(b1, b2), lj2 = dist3(b2, b0);
      if ((li0 * scale < lj0) && (lj0 < li0 / scale) && (li1 * scale < lj1) && (lj1 < li1 / scale) &&
          (li2 * scale < lj2) && (lj2 < li2 / scale))
        keep[r[0]] = keep[r[1]] = keep[r[2]] = 1;
    }
    std::vector<std::pair<int, int>> kept;
    for (i64 c = 0; c < ncorr; ++c)
      if (keep[c]) kept.push_back(corres[c]);
    corres.swap(kept);
  }
  if (swapped)
    for (auto& pr : corres) std::swap(pr.first, pr.second);
  std::sort(corres.begin(), corres.end());
  corres.erase(std::unique(corres.begin(), corres.end()), corres.end());
  if ((i64)corres.size() > capacity) return -1;
  for (size_t c = 0; c < corres.size(); ++c) {
    pairs[2 * c] = corres[c].first;
    pairs[2 * c + 1] = corres[c].second;
  }
  return (i64)corres.size();
}

// raw exact 1-NN table (kernel-level check): out[q] = argmin_i L2(query[q], db[i]), lowest index among ties
void orc_nn1(const float* query, int nq, const float* db, int ndb, int dim, int32_t* out) {
#pragma omp parallel for schedule(static)
  for (int q = 0; q < nq; ++q) out[q] = nn1(query + (size_t)q * dim, db, ndb, dim);
}

}  // extern "C"
