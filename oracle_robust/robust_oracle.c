/* robust_oracle.c -- CPU checker of the robust-kernel evaluation (vgicp_set_robust_kernel).  TEST INFRASTRUCTURE ONLY.
 *
 * The float oracle (oracle/vgicp_oracle.c) is compiled into this library unchanged, so its voxel maps, correspondence search and
 * LM loop are the ones every other test uses; this file adds the robust kind to its derivative sum (compute_derivatives_impl with
 * rho / rho') and exports a robust evaluate and a robust align.  Built with the oracle's flags (no contraction, no fast math), so
 * rho and rho' are the IEEE single operations the CUDA kernels spell (vgicp_kernels.cuh robust_rho, log_det, log1p_det).
 *   HUBER          rho = s (s <= d2), 2 sqrt(d2 s) - d2 (else)       rho' = 1, sqrt(d2 / s)
 *   CAUCHY         rho = d2 ln(1 + s / d2)                           rho' = d2 / (d2 + s)
 *   GEMAN_MCCLURE  rho = s d2 / (d2 + s)                             rho' = (d2 / (d2 + s))^2
 * err = sum w rho(s), H = sum w rho'(s) J^T M J, b = sum w rho'(s) J^T M e, w = sqrt(n_voxel).  kind 0 = the plain sums.
 */
#include "../oracle/vgicp_oracle.c"

enum { RB_NONE = 0, RB_HUBER = 1, RB_CAUCHY = 2, RB_GEMAN_MCCLURE = 3 };

static inline float f_from_bits(uint32_t u) { float f; memcpy(&f, &u, 4); return f; }
static inline uint32_t bits_from_f(float f) { uint32_t u; memcpy(&u, &f, 4); return u; }

/* ln(u), u > 0: u = m 2^k, m in [sqrt(1/2), sqrt(2)), ln m = 2 atanh((m-1)/(m+1)) by its series to f^9 (same sequence as log_det) */
static float log_det(float u) {
  if (!(u > 0.0f)) return f_from_bits(0x7fc00000u);
  if (!(u < f_from_bits(0x7f800000u))) return u;
  const uint32_t bits = bits_from_f(u);
  int k = (int)((bits >> 23) & 0xffu) - 127;
  float m = f_from_bits((bits & 0x007fffffu) | 0x3f800000u);
  if (m > 1.41421356f) {
    m = m * 0.5f;
    k += 1;
  }
  const float f = (m - 1.0f) / (m + 1.0f);
  const float f2 = f * f;
  float p = fmaf(f2, 0.111111111f, 0.142857143f);
  p = fmaf(f2, p, 0.2f);
  p = fmaf(f2, p, 0.333333333f);
  const float two_f = f + f;
  const float ln_m = fmaf(two_f * f2, p, two_f);
  const float kf = (float)k;
  return kf * 0.693359375f + fmaf(kf, -2.12194440e-4f, ln_m);
}
static float log1p_det(float x) {
  const float u = 1.0f + x;
  if (u == 1.0f) return x;
  return log_det(u) * (x / (u - 1.0f));
}
static void robust_rho(int kind, float d2, float s, float* rho, float* drho) {
  if (kind == RB_NONE) { *rho = s; *drho = 1.0f; return; }
  if (kind == RB_HUBER) {
    if (s <= d2) { *rho = s; *drho = 1.0f; }
    else {
      const float r = sqrtf(d2 * s);
      *rho = (r + r) - d2;
      *drho = sqrtf(d2 / s);
    }
    return;
  }
  const float q = d2 / (d2 + s);
  if (kind == RB_CAUCHY) { *rho = d2 * log1p_det(s / d2); *drho = q; }
  else { *rho = q * s; *drho = q * q; }
}

/* compute_derivatives_impl (VGICP, ndt = 0) with the robust terms: same per-correspondence float terms, err = w rho, and the
 * Jacobian products weighted by w rho' */
static double robust_derivatives(const OrcVoxelMap* m, const float* src, const float* src_cov9, const int* pairs, long n_pairs, const float* Tlin, const float* Teval,
                                 double* H36, double* b6, int kind, float d2) {
  double Hd[36] = {0}, bd[6] = {0}, ed = 0.0;
  int want = (H36 != NULL && b6 != NULL);
  float Rl[9], Rlt[9];
  for (int c = 0; c < 3; c++) for (int r = 0; r < 3; r++) { M3(Rl, r, c) = Tlin[c * 4 + r]; M3(Rlt, c, r) = Tlin[c * 4 + r]; }
  for (long ci = 0; ci < n_pairs; ci++) {
    int ia = pairs[2 * ci], iv = pairs[2 * ci + 1];
    if (iv < 0) continue;
    int np = m->vox_n[iv];
    if (want && np <= 0) continue;
    const float* meanA = src + 3 * (size_t)ia;
    const float* covA = src_cov9 + 9 * (size_t)ia;
    const float* meanB = m->vox_mean + 3 * (size_t)iv;
    const float* covB = m->vox_cov + 9 * (size_t)iv;
    float pa[3];
    transform_pt(Teval, meanA, pa);
    float tmp[9], RCR[9], S[9], Minv[9];
    mul3f(Rl, covA, tmp);
    mul3f(tmp, Rlt, RCR);
    for (int j = 0; j < 9; j++) S[j] = covB[j] + RCR[j];
    inv3f(S, Minv);
    float e[3] = {meanB[0] - pa[0], meanB[1] - pa[1], meanB[2] - pa[2]};
    float w = sqrtf((float)np);
    float Me[3];
    for (int r = 0; r < 3; r++) Me[r] = (M3(Minv, r, 0) * e[0] + M3(Minv, r, 1) * e[1]) + M3(Minv, r, 2) * e[2];
    float s = (e[0] * Me[0] + e[1] * Me[1]) + e[2] * Me[2];
    float rho, drho;
    robust_rho(kind, d2, s, &rho, &drho);
    ed += (double)(w * rho);
    if (!want) continue;
    float wd = kind == RB_NONE ? w : w * drho;
    float J[18]; /* column-major 3x6: J = [skew(pa) | -I] */
    memset(J, 0, sizeof(J));
    J[3 * 1 + 0] = -pa[2]; J[3 * 2 + 0] = pa[1];
    J[3 * 0 + 1] = pa[2];  J[3 * 2 + 1] = -pa[0];
    J[3 * 0 + 2] = -pa[1]; J[3 * 1 + 2] = pa[0];
    J[3 * 3 + 0] = -1.0f; J[3 * 4 + 1] = -1.0f; J[3 * 5 + 2] = -1.0f;
    float JtM[18];
    for (int r = 0; r < 6; r++)
      for (int c = 0; c < 3; c++) JtM[r * 3 + c] = ((wd * J[3 * r + 0]) * M3(Minv, 0, c) + (wd * J[3 * r + 1]) * M3(Minv, 1, c)) + (wd * J[3 * r + 2]) * M3(Minv, 2, c);
    for (int r = 0; r < 6; r++) {
      for (int c = 0; c < 6; c++) Hd[c * 6 + r] += (double)((JtM[r * 3 + 0] * J[3 * c + 0] + JtM[r * 3 + 1] * J[3 * c + 1]) + JtM[r * 3 + 2] * J[3 * c + 2]);
      bd[r] += (double)((JtM[r * 3 + 0] * e[0] + JtM[r * 3 + 1] * e[1]) + JtM[r * 3 + 2] * e[2]);
    }
  }
  if (want) {
    memcpy(H36, Hd, sizeof(Hd));
    memcpy(b6, bd, sizeof(bd));
  }
  return ed;
}

ORC_API void orc_robust_rho(int kind, float d2, const float* s, int n, float* rho, float* drho) {
  for (int i = 0; i < n; i++) robust_rho(kind, d2, s[i], rho + i, drho + i);
}

/* one evaluation: update_correspondences(Tlin) + compute_error(Teval, H, b) with the robust kind; H36 / b6 may be NULL */
ORC_API double orc_robust_evaluate_f32(const OrcVoxelMap* map, const float* src, const float* src_cov9, int n_src, const int* offsets, int n_off, const double* Tlin_d,
                                       const double* Teval_d, double* H36, double* b6, int kind, float d2, long* n_corr) {
  float Tl[16], Te[16];
  to_f32_pose(Tlin_d, Tl);
  to_f32_pose(Teval_d, Te);
  long cap = (long)n_src * n_off;
  int* pairs = (int*)malloc(sizeof(int) * 2 * (size_t)(cap > 0 ? cap : 1));
  long np = orc_find_correspondences(map, src, n_src, Tl, offsets, n_off, pairs, cap);
  double e = robust_derivatives(map, src, src_cov9, pairs, np, Tl, Te, H36, b6, kind, d2);
  if (n_corr) *n_corr = np;
  free(pairs);
  return e;
}

/* the derivatives at Teval over a caller-given correspondence list (fixed correspondences and linearisation pose) */
ORC_API double orc_robust_derivatives(const OrcVoxelMap* map, const float* src, const float* src_cov9, const int* pairs, long n_pairs, const double* Tlin_d,
                                      const double* Teval_d, double* H36, double* b6, int kind, float d2) {
  float Tl[16], Te[16];
  to_f32_pose(Tlin_d, Tl);
  to_f32_pose(Teval_d, Te);
  return robust_derivatives(map, src, src_cov9, pairs, n_pairs, Tl, Te, H36, b6, kind, d2);
}

typedef struct {
  F32Problem p;
  int kind;
  float d2;
} RobustProblem;

static double robust_linearize(void* c, const double* T, double* H, double* b) {
  RobustProblem* r = (RobustProblem*)c;
  F32Problem* p = &r->p;
  to_f32_pose(T, p->Tlin);
  p->n_pairs = orc_find_correspondences(p->map, p->src, p->n_src, p->Tlin, p->offsets, p->n_off, p->pairs, p->cap_pairs);
  float Te[16];
  to_f32_pose(T, Te);
  return robust_derivatives(p->map, p->src, p->src_cov9, p->pairs, p->n_pairs, p->Tlin, Te, H, b, r->kind, r->d2);
}
static double robust_error(void* c, const double* T) {
  RobustProblem* r = (RobustProblem*)c;
  F32Problem* p = &r->p;
  float Te[16];
  to_f32_pose(T, Te);
  return robust_derivatives(p->map, p->src, p->src_cov9, p->pairs, p->n_pairs, p->Tlin, Te, NULL, NULL, r->kind, r->d2);
}

/* orc_align_f32 (double sums) with the robust kind */
ORC_API int orc_robust_align_f32(const OrcVoxelMap* map, const float* src, const float* src_cov9, int n_src, const int* offsets, int n_off, const OrcLsqParams* params,
                                 const double* guess, int kind, float d2, OrcLsqResult* res) {
  RobustProblem r;
  memset(&r, 0, sizeof(r));
  r.p.map = map; r.p.src = src; r.p.src_cov9 = src_cov9; r.p.n_src = n_src; r.p.offsets = offsets; r.p.n_off = n_off;
  r.p.cap_pairs = (long)n_src * n_off;
  r.p.pairs = (int*)malloc(sizeof(int) * 2 * (size_t)(r.p.cap_pairs > 0 ? r.p.cap_pairs : 1));
  r.kind = kind; r.d2 = d2;
  lsq_optimize(params, &r, robust_linearize, robust_error, guess, res);
  free(r.p.pairs);
  return 0;
}
