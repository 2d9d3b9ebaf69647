// Voxel-grid downsampling (the first step of the reference's FPFH + TEASER++ + ICP tutorial, DESIGN.md §3.12):
// Open3D's PointCloud::VoxelDownSample, points and optionally colours, with the output order and the non-finite rule that
// include/teaser_b200.h defines, for B clouds stored back to back.
//
//   vox_bounds_kernel  per point: component-wise min / max of each cloud's finite points (ordered-int float atomics)
//   vox_setup_kernel   per cloud: vmin, Open3D's INT_MAX check, the per-axis voxel counts and the 2^62-cell limit
//   vox_key_kernel     per point: its voxel key (i_x c_y + i_y) c_z + i_z, or kVoxNone when it belongs to no voxel
//   CUB radix sort     (key, point) pairs over the whole batch, stable
//   vox_cloud_kernel   per sorted point: its cloud
//   CUB radix sort     (cloud, point) pairs, stable: points grouped by (cloud, key), each group ascending by index
//   vox_head_kernel    per sorted point: marks the first member of every voxel (by input index) and the group bounds
//   CUB exclusive sum  of those marks in input order: each voxel's output row, ordered by its first member
//   vox_mean_kernel    per voxel: the sequential float64 sum of its members in ascending index, the mean, voxel_of
//                      (<true>: also the members' colours, tzr_voxel_downsample_colors)
//   vox_count_kernel   per cloud: its first output row and its number of voxels
//
// Ten launches whatever B.  Every per-cloud quantity depends on the cloud's own points only, so a cloud's outputs do not
// depend on the batch it runs in.
#include <cub/cub.cuh>

#include <algorithm>

#include "tzr_internal.cuh"

namespace tzr {

namespace {

constexpr int kVoxThreads = 256;

__device__ __forceinline__ int vox_cloud_of(const VoxCloud* __restrict__ cl, int B, int i) {
  int lo = 0, hi = B - 1;  // the last cloud whose first point is <= i (every cloud holds at least one point)
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (cl[mid].lo <= i) lo = mid;
    else hi = mid - 1;
  }
  return lo;
}

__device__ __forceinline__ bool vox_finite(const float* __restrict__ pts, int i) {
  return isfinite(pts[3 * (size_t)i]) && isfinite(pts[3 * (size_t)i + 1]) && isfinite(pts[3 * (size_t)i + 2]);
}

// per-cloud bounds of the finite points; a warp whose lanes share one cloud reduces before its atomics
__global__ void vox_bounds_kernel(const float* __restrict__ pts, int N, VoxCloud* cl, int B) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  int mn[3] = {0x7fffffff, 0x7fffffff, 0x7fffffff};
  int mx[3] = {(int)0x80000000, (int)0x80000000, (int)0x80000000};
  int c = -1;
  if (i < N) {
    c = vox_cloud_of(cl, B, i);
    if (vox_finite(pts, i))
      for (int k = 0; k < 3; ++k) mn[k] = mx[k] = f2ord(pts[3 * (size_t)i + k]);
  }
  const bool uniform = __all_sync(0xffffffffu, c == __shfl_sync(0xffffffffu, c, 0));
  for (int k = 0; k < 3; ++k) {
    if (uniform)
      for (int off = 16; off; off >>= 1) {
        mn[k] = min(mn[k], __shfl_xor_sync(0xffffffffu, mn[k], off));
        mx[k] = max(mx[k], __shfl_xor_sync(0xffffffffu, mx[k], off));
      }
    if ((!uniform || (threadIdx.x & 31) == 0) && mn[k] != 0x7fffffff) {
      atomicMin(&cl[c].mn[k], mn[k]);
      atomicMax(&cl[c].mx[k], mx[k]);
    }
  }
}

// Open3D's bounds and its INT_MAX check, then the grid: axis k has c_k = i_k(max_k) + 1 voxels, the index of the
// largest finite coordinate computed exactly as every point's index is (rounding is monotone, so every finite point
// of the cloud has 0 <= i_k < c_k).  The key (i_x c_y + i_y) c_z + i_z is below c_x c_y c_z <= 2^62.
__global__ void vox_setup_kernel(VoxCloud* cl, int B, double v) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= B) return;
  VoxCloud& c = cl[b];
  c.status = TZR_OK;
  c.valid = 0;
  c.cy = c.cz = 1;
  if (c.mn[0] == 0x7fffffff) return;  // no finite point: no voxel
  const double h = __dmul_rn(v, 0.5);
  double hi[3], ext = 0.0;
  for (int k = 0; k < 3; ++k) {
    hi[k] = (double)ord2f(c.mx[k]);
    c.vmin[k] = __dsub_rn((double)ord2f(c.mn[k]), h);
    const double vmax = __dadd_rn(hi[k], h);
    ext = fmax(ext, __dsub_rn(vmax, c.vmin[k]));
  }
  if (__dmul_rn(v, 2147483647.0) < ext) {  // voxel_size * INT_MAX < (vmax - vmin).maxCoeff()
    c.status = TZR_ERR_TOO_LARGE;
    return;
  }
  unsigned long long cnt[3];
  for (int k = 0; k < 3; ++k) cnt[k] = (unsigned long long)(int)floor(__ddiv_rn(__dsub_rn(hi[k], c.vmin[k]), v)) + 1ull;
  const unsigned long long lim = 1ull << 62;
  const unsigned long long xy = cnt[0] * cnt[1];  // each count is at most 2^31: no overflow
  if (xy > lim || cnt[2] > lim / xy) {
    c.status = TZR_ERR_TOO_LARGE;
    return;
  }
  c.cy = (long long)cnt[1];
  c.cz = (long long)cnt[2];
  c.valid = 1;
}

// i_k = (int) floor((p_k - vmin_k) / v): a division, as Open3D writes it (a product with 1/v differs on voxel edges)
__global__ void vox_key_kernel(const float* __restrict__ pts, int N, const VoxCloud* __restrict__ cl, int B, double v,
                               unsigned long long* __restrict__ key, int* __restrict__ idx) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= N) return;
  idx[i] = i;
  const VoxCloud& c = cl[vox_cloud_of(cl, B, i)];
  unsigned long long k = kVoxNone;
  if (c.valid && vox_finite(pts, i)) {
    long long ix[3];
    for (int a = 0; a < 3; ++a)
      ix[a] = (int)floor(__ddiv_rn(__dsub_rn((double)pts[3 * (size_t)i + a], c.vmin[a]), v));
    k = (unsigned long long)((ix[0] * c.cy + ix[1]) * c.cz + ix[2]);
  }
  key[i] = k;
}

__global__ void vox_cloud_kernel(const int* __restrict__ idx, int N, const VoxCloud* __restrict__ cl, int B,
                                 unsigned int* __restrict__ cloud) {
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r < N) cloud[r] = (unsigned int)vox_cloud_of(cl, B, idx[r]);
}

// In sorted order (cloud, key, index): mark[r] = 1 where a voxel starts, 2 for a point in no voxel (each such point
// is a group of its own), 0 inside a voxel; head[i] = 1 for the first (lowest-index) member of a voxel
__global__ void vox_head_kernel(const int* __restrict__ idx, const unsigned int* __restrict__ cloud,
                                const unsigned long long* __restrict__ key, int N, unsigned char* __restrict__ mark,
                                int* __restrict__ head) {
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= N) return;
  const int i = idx[r];
  const unsigned long long k = key[i];
  int f = 0;
  if (k == kVoxNone) f = 2;
  else if (r == 0 || cloud[r - 1] != cloud[r] || key[idx[r - 1]] != k) f = 1;
  mark[r] = (unsigned char)f;
  head[i] = f == 1;
}

// One thread per voxel: its members are the sorted positions [r, e) up to the next mark, ascending by input index; the
// sum starts at 0.0 and adds them one at a time (Open3D's AccumulatedPoint), the mean is rounded once to float.
// kColors (tzr_voxel_downsample_colors, DESIGN.md §3.17): the members' colours are averaged the same way into
// colors_out; the instance without it ignores both pointers.
template <bool kColors>
__global__ void __launch_bounds__(kVoxThreads) vox_mean_kernel(const float* __restrict__ pts, const int* __restrict__ idx,
                                                               const unsigned int* __restrict__ cloud,
                                                               const unsigned char* __restrict__ mark,
                                                               const int* __restrict__ row, int N,
                                                               const VoxCloud* __restrict__ cl,
                                                               float* __restrict__ out, int* __restrict__ voxel_of,
                                                               const float* __restrict__ colors,
                                                               float* __restrict__ colors_out) {
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= N) return;
  const int f = mark[r];
  if (f == 0) return;
  const int i = idx[r];
  if (f == 2) {
    voxel_of[i] = -1;
    return;
  }
  const int g = row[i];                       // output row in the batch
  const int local = g - row[cl[cloud[r]].lo];  // ... and in its cloud
  int e = r + 1;
  while (e < N && mark[e] == 0) ++e;
  double s0 = 0.0, s1 = 0.0, s2 = 0.0;
#pragma unroll 4
  for (int q = r; q < e; ++q) {
    const size_t j = (size_t)idx[q];
    s0 = __dadd_rn(s0, (double)pts[3 * j]);
    s1 = __dadd_rn(s1, (double)pts[3 * j + 1]);
    s2 = __dadd_rn(s2, (double)pts[3 * j + 2]);
    voxel_of[j] = local;
  }
  const double cnt = (double)(e - r);
  out[3 * (size_t)g] = __double2float_rn(__ddiv_rn(s0, cnt));
  out[3 * (size_t)g + 1] = __double2float_rn(__ddiv_rn(s1, cnt));
  out[3 * (size_t)g + 2] = __double2float_rn(__ddiv_rn(s2, cnt));
  if constexpr (kColors) {
    double c0 = 0.0, c1 = 0.0, c2 = 0.0;
    for (int q = r; q < e; ++q) {
      const size_t j = (size_t)idx[q];
      c0 = __dadd_rn(c0, (double)colors[3 * j]);
      c1 = __dadd_rn(c1, (double)colors[3 * j + 1]);
      c2 = __dadd_rn(c2, (double)colors[3 * j + 2]);
    }
    colors_out[3 * (size_t)g] = __double2float_rn(__ddiv_rn(c0, cnt));
    colors_out[3 * (size_t)g + 1] = __double2float_rn(__ddiv_rn(c1, cnt));
    colors_out[3 * (size_t)g + 2] = __double2float_rn(__ddiv_rn(c2, cnt));
  }
}

__global__ void vox_count_kernel(const int* __restrict__ head, const int* __restrict__ row, VoxCloud* cl, int B) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= B) return;
  VoxCloud& c = cl[b];
  const int last = c.lo + c.n - 1;
  c.out_lo = row[c.lo];
  c.n_out = row[last] + head[last] - row[c.lo];
}

int bits_for(unsigned int v) {  // bits that hold 0 ... v
  int bits = 1;
  while (bits < 32 && (1ull << bits) <= v) ++bits;
  return bits;
}

struct VoxScratch {
  unsigned long long *key, *key2;
  int *idx, *idx1, *idx2, *head, *row;
  unsigned int *cloud1, *cloud2;
  unsigned char* mark;
  void* cub;
  size_t cub_bytes;
};

// carves the scratch of N points; with base == nullptr only the sizes are computed
size_t vox_carve(int N, int B, char* base, VoxScratch* s) {
  size_t cub_bytes = 0, t = 0;
  cub::DeviceRadixSort::SortPairs(nullptr, t, (const unsigned long long*)nullptr, (unsigned long long*)nullptr,
                                  (const int*)nullptr, (int*)nullptr, N, 0, kVoxKeyBits);
  cub_bytes = std::max(cub_bytes, t);
  cub::DeviceRadixSort::SortPairs(nullptr, t, (const unsigned int*)nullptr, (unsigned int*)nullptr,
                                  (const int*)nullptr, (int*)nullptr, N, 0, bits_for((unsigned int)(B - 1)));
  cub_bytes = std::max(cub_bytes, t);
  cub::DeviceScan::ExclusiveSum(nullptr, t, (const int*)nullptr, (int*)nullptr, N);
  cub_bytes = std::max(cub_bytes, t);
  size_t off = 0;
  auto take = [&](size_t bytes) {
    char* p = base ? base + off : nullptr;
    off += (bytes + 255) & ~(size_t)255;
    return p;
  };
  const size_t n = (size_t)N;
  s->key = (unsigned long long*)take(n * 8);
  s->key2 = (unsigned long long*)take(n * 8);
  s->idx = (int*)take(n * 4);
  s->idx1 = (int*)take(n * 4);
  s->idx2 = (int*)take(n * 4);
  s->head = (int*)take(n * 4);
  s->row = (int*)take(n * 4);
  s->cloud1 = (unsigned int*)take(n * 4);
  s->cloud2 = (unsigned int*)take(n * 4);
  s->mark = (unsigned char*)take(n);
  s->cub = take(cub_bytes);
  s->cub_bytes = cub_bytes;
  return off;
}

}  // namespace

int voxel_plan(int B, const int32_t* n, VoxCloud* clouds, VoxPlan* plan) {
  long long lo = 0;
  for (int b = 0; b < B; ++b) {
    VoxCloud& c = clouds[b];
    c = VoxCloud{};
    c.lo = (int)lo;
    c.n = n[b];
    for (int k = 0; k < 3; ++k) {
      c.mn[k] = 0x7fffffff;
      c.mx[k] = (int)0x80000000;
    }
    lo += n[b];
    if (lo > 0x7fffffffll) return TZR_ERR_TOO_LARGE;
  }
  plan->B = B;
  plan->N = (int)lo;
  VoxScratch s;
  plan->scratch_bytes = vox_carve(plan->N, B, nullptr, &s);
  return TZR_OK;
}

int launch_voxel(const VoxPlan& plan, double voxel_size, const float* pts, VoxCloud* clouds, void* scratch, float* out,
                 int* voxel_of, cudaStream_t st, const float* colors, float* colors_out) {
  const int N = plan.N, B = plan.B;
  VoxScratch s;
  vox_carve(N, B, (char*)scratch, &s);
  const int gp = (N + kVoxThreads - 1) / kVoxThreads, gc = (B + 127) / 128;
  vox_bounds_kernel<<<gp, kVoxThreads, 0, st>>>(pts, N, clouds, B);
  vox_setup_kernel<<<gc, 128, 0, st>>>(clouds, B, voxel_size);
  vox_key_kernel<<<gp, kVoxThreads, 0, st>>>(pts, N, clouds, B, voxel_size, s.key, s.idx);
  size_t t = s.cub_bytes;
  cub::DeviceRadixSort::SortPairs(s.cub, t, s.key, s.key2, s.idx, s.idx1, N, 0, kVoxKeyBits, st);
  vox_cloud_kernel<<<gp, kVoxThreads, 0, st>>>(s.idx1, N, clouds, B, s.cloud1);
  t = s.cub_bytes;
  cub::DeviceRadixSort::SortPairs(s.cub, t, s.cloud1, s.cloud2, s.idx1, s.idx2, N, 0,
                                  bits_for((unsigned int)(B - 1)), st);
  vox_head_kernel<<<gp, kVoxThreads, 0, st>>>(s.idx2, s.cloud2, s.key, N, s.mark, s.head);
  t = s.cub_bytes;
  cub::DeviceScan::ExclusiveSum(s.cub, t, s.head, s.row, N, st);
  if (colors)
    vox_mean_kernel<true><<<gp, kVoxThreads, 0, st>>>(pts, s.idx2, s.cloud2, s.mark, s.row, N, clouds, out, voxel_of,
                                                        colors, colors_out);
  else
    vox_mean_kernel<false><<<gp, kVoxThreads, 0, st>>>(pts, s.idx2, s.cloud2, s.mark, s.row, N, clouds, out, voxel_of,
                                                         nullptr, nullptr);
  vox_count_kernel<<<gc, 128, 0, st>>>(s.head, s.row, clouds, B);
  return 10;
}

// One CTA per cloud: its points through its pose in float64 (each product and sum rounded on its own, so the result
// does not depend on contraction), rounded once to float; its colours copied alongside.
__global__ void __launch_bounds__(256) map_transform_kernel(const MapCloud* __restrict__ clouds,
                                                            const float* __restrict__ pts,
                                                            const float* __restrict__ colors, float* __restrict__ out,
                                                            float* __restrict__ colors_out) {
  const MapCloud c = clouds[blockIdx.x];
  for (int i = threadIdx.x; i < c.n; i += blockDim.x) {
    const size_t s = 3 * ((size_t)c.src_lo + i), d = 3 * ((size_t)c.dst_lo + i);
    const double x = pts[s], y = pts[s + 1], z = pts[s + 2];
#pragma unroll
    for (int r = 0; r < 3; ++r)
      out[d + r] = (float)__dadd_rn(
          __dadd_rn(__dadd_rn(__dmul_rn(c.T[3 * r], x), __dmul_rn(c.T[3 * r + 1], y)), __dmul_rn(c.T[3 * r + 2], z)),
          c.T[9 + r]);
    if (colors) {
      colors_out[d] = colors[s];
      colors_out[d + 1] = colors[s + 1];
      colors_out[d + 2] = colors[s + 2];
    }
  }
}

int launch_map_transform(const MapCloud* clouds, int n_clouds, const float* pts, const float* colors, float* out,
                         float* colors_out, cudaStream_t st) {
  map_transform_kernel<<<n_clouds, 256, 0, st>>>(clouds, pts, colors, out, colors_out);
  return 1;
}

}  // namespace tzr
