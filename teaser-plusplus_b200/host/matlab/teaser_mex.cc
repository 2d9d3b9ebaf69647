// MATLAB MEX entry point `teaser_solve_mex` for the GPU path — same positional contract as the reference's
// matlab/teaser_mex.cc:19-38,99-244:
//   [s, R, t, time_ms] = teaser_solve_mex(src(3xN), dst(3xN), cbar2, noise_bound, estimate_scaling(logical),
//                                         rot_alg(0 GNC_TLS | 1 FGR | 2 QUATRO), rotation_gnc_factor,
//                                         rotation_max_iterations, rotation_cost_threshold,
//                                         inlier_selection_algorithm(0 PMC_EXACT | 1 PMC_HEU | 2 KCORE_HEU | 3 NONE),
//                                         kcore_heuristic_threshold)
// MATLAB 3xN doubles are column-major, i.e. already in the C-ABI layout: the arrays are passed straight through.
// Build inside MATLAB:  mex -I<repo>/include teaser_mex.cc -L<repo>/teaser-plusplus_b200/csrc -lteaser_b200
// (MATLAB is not part of this image; tests/test_facade_cpu.py compiles this file against mex_stub.h for syntax.)
#include <chrono>
#include <cstring>

#ifdef TZR_MEX_SYNTAX_CHECK
#include "mex_stub.h"
#else
#include "mex.h"
#endif

#include "teaser_b200.h"

namespace {
tzr_ctx* g_ctx = nullptr;
void release_ctx() {
  if (g_ctx) tzr_ctx_destroy(g_ctx);
  g_ctx = nullptr;
}
bool is_real_double_scalar(const mxArray* a) {
  return mxIsDouble(a) && !mxIsComplex(a) && mxGetNumberOfElements(a) == 1;
}
bool is_point_cloud(const mxArray* a) { return mxIsDouble(a) && !mxIsComplex(a) && mxGetM(a) == 3; }
}  // namespace

void mexFunction(int nlhs, mxArray* plhs[], int nrhs, const mxArray* prhs[]) {
  if (nrhs != 11) mexErrMsgIdAndTxt("teaserSolve:nargin", "Wrong number of input arguments (expected 11).");
  if (nlhs != 4) mexErrMsgIdAndTxt("teaserSolve:nargout", "Wrong number of output arguments (expected 4).");
  if (!is_point_cloud(prhs[0]) || !is_point_cloud(prhs[1]) || mxGetN(prhs[0]) != mxGetN(prhs[1]))
    mexErrMsgIdAndTxt("teaserSolve:inputType", "src and dst must be real double 3-by-N matrices of equal size.");
  for (int k = 2; k < 11; ++k) {
    if (k == 4) {
      if (!mxIsLogicalScalar(prhs[k])) mexErrMsgIdAndTxt("teaserSolve:inputType", "estimate_scaling must be logical.");
    } else if (!is_real_double_scalar(prhs[k])) {
      mexErrMsgIdAndTxt("teaserSolve:inputType", "Scalar parameters must be real doubles.");
    }
  }
  if (!g_ctx) {
    if (tzr_ctx_create(-1, &g_ctx) != TZR_OK)
      mexErrMsgIdAndTxt("teaserSolve:noDevice", "No usable CUDA device (the GPU path has no CPU fallback).");
    mexAtExit(release_ctx);
  }
  tzr_params p;
  tzr_params_default(&p);
  p.cbar2 = *mxGetPr(prhs[2]);
  p.noise_bound = *mxGetPr(prhs[3]);
  p.estimate_scaling = mxIsLogicalScalarTrue(prhs[4]) ? 1 : 0;
  const int rot = static_cast<int>(*mxGetPr(prhs[5]));
  p.rotation_estimation_algorithm = (rot >= 0 && rot <= 2) ? rot : 0;  // unknown -> GNC_TLS (teaser_mex.cc:170-173)
  p.rotation_gnc_factor = *mxGetPr(prhs[6]);
  p.rotation_max_iterations = static_cast<uint64_t>(*mxGetPr(prhs[7]));
  p.rotation_cost_threshold = *mxGetPr(prhs[8]);
  const int sel = static_cast<int>(*mxGetPr(prhs[9]));
  p.inlier_selection_mode = (sel >= 0 && sel <= 3) ? sel : 0;  // unknown -> PMC_EXACT (teaser_mex.cc:201-204)
  p.kcore_heuristic_threshold = *mxGetPr(prhs[10]);

  const int n = static_cast<int>(mxGetN(prhs[0]));
  tzr_solution s;
  const auto t0 = std::chrono::high_resolution_clock::now();
  const int rc = tzr_solve(g_ctx, &p, mxGetPr(prhs[0]), mxGetPr(prhs[1]), n, &s, nullptr, nullptr, nullptr);
  const auto t1 = std::chrono::high_resolution_clock::now();
  if (rc != TZR_OK) mexErrMsgIdAndTxt("teaserSolve:solve", tzr_status_string(rc));
  plhs[0] = mxCreateDoubleScalar(s.scale);
  plhs[1] = mxCreateDoubleMatrix(3, 3, mxREAL);
  std::memcpy(mxGetPr(plhs[1]), s.rotation, sizeof(s.rotation));  // both column-major
  plhs[2] = mxCreateDoubleMatrix(3, 1, mxREAL);
  std::memcpy(mxGetPr(plhs[2]), s.translation, sizeof(s.translation));
  plhs[3] = mxCreateDoubleScalar(std::chrono::duration<double, std::milli>(t1 - t0).count());
}
