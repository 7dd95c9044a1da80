// EKF kernels (HOT LOOPs 2-4 of SURVEY.md §3.2): per-feature Jacobian + Mahalanobis gate,
// measurement update, covariance slot surgery, propagation strips, depth sub-filter, OOS
// projection.  All fp64 (the reference is fp64 Eigen, /root/reference/common/alias.h:11);
// the covariance P stays resident in HBM, one N x N block per independent filter.
#include "hostmath.h"
#include <atomic>
#include <algorithm>

#include "kernels.h"
#include "prof.h"

namespace xb {

__device__ __forceinline__ double warp_sum_d(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// ------------------------------------------------------------------------------------------
// Jacobian + gate.  One warp per in-state feature.
// Follows Feature::ComputeJacobian (/root/reference/src/feature.cpp:542-656) for the chain
// x -> Xc -> Xbr -> Xs -> Xb -> Xcn -> xcn -> xp and the MH distance of Estimator::MHGating
// (/root/reference/src/update.cpp:60-69), exploiting that J has only 21 non-zero columns
// (the reference multiplies the full 2xN by NxN).
// ------------------------------------------------------------------------------------------
__device__ void compute_feature_jacobian(const EkfLayout lay, const CameraParams& cam, const double* X, const double* grp,
                                         const double* x, const double* xp, int ref_sind, int f_sind, FeatJac* o) {
  M3 Rsb, Rbc, Rr;
  V3 Tsb, Tbc, Tr;
  for (int i = 0; i < 9; ++i) { Rsb.m[i] = X[i]; Rbc.m[i] = X[12 + i]; Rr.m[i] = grp[i]; }
  for (int i = 0; i < 3; ++i) { Tsb.v[i] = X[9 + i]; Tbc.v[i] = X[21 + i]; Tr.v[i] = grp[9 + i]; }
  const M3 Rsb_t = m3_t(Rsb), Rbc_t = m3_t(Rbc);
  // unproject_logz (/root/reference/common/project.h:79-95)
  const double z = exp(x[2]);
  const V3 Xc{{x[0] * z, x[1] * z, z}};
  const M3 dXc_dx{{z, 0, x[0] * z, 0, z, x[1] * z, 0, 0, z}};
  const V3 Xbr = v3_add(m3_mulv(Rbc, Xc), Tbc);
  const V3 Xs = v3_add(m3_mulv(Rr, Xbr), Tr);
  const V3 Xb = m3_mulv(Rsb_t, v3_sub(Xs, Tsb));
  const V3 Xcn = m3_mulv(Rbc_t, v3_sub(Xb, Tbc));
  const M3 A = m3_mul(Rbc_t, Rsb_t);  // dXcn_dXs
  const M3 B = m3_mul(A, Rr);         // dXcn_dXbr
  const M3 dXcn_dTbc = m3_add(m3_neg(Rbc_t), B);
  const M3 dXcn_dWbc = m3_add(m3_hat(Xcn), m3_mul(B, m3_neg(m3_mul(Rbc, m3_hat(Xc)))));
  const M3 dXcn_dTsb = m3_neg(A);
  const M3 dXcn_dWsb = m3_mul(Rbc_t, m3_hat(Xb));
  const M3 dXcn_dTsbr = A;
  const M3 dXcn_dWsbr = m3_mul(A, m3_neg(m3_mul(Rr, m3_hat(Xbr))));
  const M3 dXcn_dx = m3_mul(m3_mul(B, Rbc), dXc_dx);
  // project (/root/reference/common/project.h:11-24)
  const double iz = 1.0 / Xcn.v[2];
  const double xcn0 = Xcn.v[0] * iz, xcn1 = Xcn.v[1] * iz;
  const double P23[6] = {iz, 0, -Xcn.v[0] * iz * iz, 0, iz, -Xcn.v[1] * iz * iz};
  double u, v, Jc[4];
  camera_project(cam, xcn0, xcn1, &u, &v, Jc);
  M23 d;
  for (int j = 0; j < 3; ++j) {
    d.m[j] = Jc[0] * P23[j] + Jc[1] * P23[3 + j];
    d.m[3 + j] = Jc[2] * P23[j] + Jc[3] * P23[3 + j];
  }
  const M3* blocks[7] = {&dXcn_dWsb, &dXcn_dTsb, &dXcn_dWbc, &dXcn_dTbc, &dXcn_dWsbr, &dXcn_dTsbr, &dXcn_dx};
  for (int b = 0; b < 7; ++b) {
    const M23 jb = m23_mul(d, *blocks[b]);
    for (int j = 0; j < 3; ++j) {
      o->J[0][3 * b + j] = jb.m[j];
      o->J[1][3 * b + j] = jb.m[3 + j];
    }
  }
  o->inn[0] = xp[0] - u;
  o->inn[1] = xp[1] - v;
  o->goff = lay.goff(ref_sind);
  o->foff = lay.foff(f_sind);
}

__device__ __forceinline__ int jac_col(int k, int goff, int foff) {
  // compact column k (0..20) -> error-state column
  return k < 6 ? k : (k < 12 ? 15 + (k - 6) : (k < 18 ? goff + (k - 12) : foff + (k - 18)));
}

// The covariance edit list of one filter (AddGroupToState / AddFeatureToState / Remove* / FixFeatureXY / SwitchRefGroup,
// /root/reference/src/estimator.cpp:739-846, :1362-1391, :1474-1478), applied in order by the whole CTA.  cov_edit_kernel is this
// function alone; the Jacobian / gate kernel and the gain kernel call it first, so that the edits that precede them cost no launch.
__device__ __forceinline__ void apply_edits(int N, double* __restrict__ Pb, const EditOp* __restrict__ ops, int n, int tid, int nthr) {
  for (int o = 0; o < n; ++o) {
    const EditOp op = ops[o];
    if (op.type == 0) {
      for (int t = tid; t < op.n * N; t += nthr) {
        const int r = t / N, c = t - r * N;
        Pb[(size_t)(op.a + r) * N + c] = 0.0;
        Pb[(size_t)c * N + op.a + r] = 0.0;
      }
    } else if (op.type == 1) {
      for (int t = tid; t < op.n * N; t += nthr) {  // rows: P[a+r, :] = P[b+r, :]
        const int r = t / N, c = t - r * N;
        Pb[(size_t)(op.a + r) * N + c] = Pb[(size_t)(op.b + r) * N + c];
      }
      __syncthreads();
      for (int t = tid; t < op.n * N; t += nthr) {  // cols: P[:, a+r] = P[:, b+r]
        const int r = t / N, c = t - r * N;
        Pb[(size_t)c * N + op.a + r] = Pb[(size_t)c * N + op.b + r];
      }
    } else if (op.type == 2) {
      if (tid < 9) Pb[(size_t)(op.a + tid / 3) * N + op.a + tid % 3] = op.blk[tid];
    }
    __syncthreads();
  }
}

// One CTA per filter: [edit list] -> one warp per in-state feature (Jacobian on lane 0, the 21 x 21 gate contraction over the lanes).
constexpr int JG_MAX_WARPS = 16;
__global__ void __launch_bounds__(JG_MAX_WARPS * 32) jacobian_gate_kernel(EkfLayout lay, const CameraParams* __restrict__ cam,
                                                           const double* __restrict__ X, const double* __restrict__ groups,
                                                           const double* __restrict__ feat_x, const double* __restrict__ feat_xp,
                                                           const int* __restrict__ feat_ref, const int* __restrict__ feat_sind,
                                                           const int* __restrict__ nfeat, double* __restrict__ P,
                                                           const double* __restrict__ Rmeas, FeatJac* __restrict__ out,
                                                           double* __restrict__ J_dense, double* __restrict__ mh_out,
                                                           const EditOp* __restrict__ ops, const int* __restrict__ ops_first,
                                                           const int* __restrict__ nops, double* __restrict__ diag_out) {
  const int b = blockIdx.x, lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
  const int N = lay.N();
  double* __restrict__ Pb = P + (size_t)b * N * N;
  if (ops) apply_edits(N, Pb, ops + ops_first[b], nops[b], threadIdx.x, blockDim.x);  // uniform over the CTA (barriers inside)
  if (diag_out)  // diagonal of P after this frame's edits (FindNewRefGroup of the 1-point RANSAC reads it on the host)
    for (int i = threadIdx.x; i < N; i += blockDim.x) diag_out[(size_t)b * N + i] = Pb[(size_t)i * N + i];
  __shared__ FeatJac sjs[JG_MAX_WARPS];
  FeatJac& sj = sjs[warp];
  const int nf = nfeat[b];
  for (int i = warp; i < nf; i += nwarps) {
  const size_t fi = (size_t)b * lay.F + i;
  __syncwarp();
  if (lane == 0) {
    const int ref = feat_ref[fi];
    compute_feature_jacobian(lay, cam[b], X + (size_t)b * kPoseDoubles, groups + ((size_t)b * lay.G + ref) * kGroupDoubles,
                             feat_x + 3 * fi, feat_xp + 2 * fi, ref, feat_sind[fi], &sj);
  }
  __syncwarp();
  const int goff = sj.goff, foff = sj.foff;
  double s00 = 0, s01 = 0, s11 = 0;
  for (int t = lane; t < kJacNnz * kJacNnz; t += 32) {
    const int a = t / kJacNnz, c = t - a * kJacNnz;
    const double p = Pb[(size_t)jac_col(a, goff, foff) * N + jac_col(c, goff, foff)];
    const double j0a = sj.J[0][a], j1a = sj.J[1][a];
    s00 += j0a * p * sj.J[0][c];
    s01 += j0a * p * sj.J[1][c];
    s11 += j1a * p * sj.J[1][c];
  }
  s00 = warp_sum_d(s00);
  s01 = warp_sum_d(s01);
  s11 = warp_sum_d(s11);
  const double R = Rmeas[b];
  s00 += R;
  s11 += R;
  const double r0 = sj.inn[0], r1 = sj.inn[1];
  const double mh = (r0 * r0 * s11 - 2.0 * r0 * r1 * s01 + r1 * r1 * s00) / (s00 * s11 - s01 * s01);
  if (lane == 0) {
    sj.mh = mh;
    out[fi] = sj;
    if (mh_out) mh_out[fi] = mh;
  }
  if (J_dense) {
    // coalesced zero fill of the two dense rows, then the 42 non-zeros
    double* __restrict__ Jd = J_dense + fi * 2 * (size_t)N;
    for (int c = lane; c < 2 * N; c += 32) Jd[c] = 0.0;
    __syncwarp();
    for (int t = lane; t < 2 * kJacNnz; t += 32) {
      const int r = t / kJacNnz, k = t - r * kJacNnz;
      Jd[(size_t)r * N + jac_col(k, goff, foff)] = sj.J[r][k];
    }
  }
  }  // features of this warp
}

int launch_jacobian_gate(cudaStream_t st, EkfLayout lay, const CameraParams* cam, const double* X, const double* groups,
                         const double* feat_x, const double* feat_xp, const int* feat_ref, const int* feat_sind,
                         const int* nfeat, double* P, const double* Rmeas, FeatJac* out, double* J_dense, double* mh_out,
                         int batch, const EditOp* ops, const int* ops_first, const int* nops, double* diag_out) {
  ProfScope ps("jacobian_gate", st);
  const int warps = std::max(1, std::min(lay.F, JG_MAX_WARPS));
  jacobian_gate_kernel<<<batch, warps * 32, 0, st>>>(lay, cam, X, groups, feat_x, feat_xp, feat_ref, feat_sind, nfeat, P, Rmeas, out,
                                                     J_dense, mh_out, ops, ops_first, nops, diag_out);
  XB_CUDA(cudaGetLastError());
  return 0;
}

// ------------------------------------------------------------------------------------------
// Measurement update.
// Reference: Estimator::FilterUpdate + UpdateJosephForm (/root/reference/src/update.cpp:120-153,
// /root/reference/src/estimator.cpp:1257-1288): S = H P H^T + R, K^T = S^-1 (H P), err = K inn,
// P <- (KH-I) P (KH-I)^T + K R K^T.
// Here: gain kernel (one CTA per filter) forms HP from the 18 non-zeros per row of H
// (FillJacobianBlock layout incl. its group-rotation quirk, feature.cpp:675-676), S, Cholesky of
// S in shared memory, K^T by substitution; covariance kernel (upper-triangle 32x32 tiles over
// all SMs) applies P <- P - K (H P) with the result mirrored so P stays exactly symmetric.
// Algebra: for the optimal gain Joseph's form equals P - K H P exactly; expanding Joseph gives
// P - K HP + K^T-side term K (S K^T - H P) whose bracket is the solve residual (~1e-16 |HP|).
// ------------------------------------------------------------------------------------------
constexpr int GAIN_THREADS = 512;
constexpr int kHnnz = 21;

template <bool SPARSE>
__global__ void __launch_bounds__(GAIN_THREADS) ekf_gain_kernel(int N, EkfLayout lay, const FeatJac* __restrict__ jac,
                                                                const int* __restrict__ sel, const int* __restrict__ nsel,
                                                                int Mdense, const double* __restrict__ Hd,
                                                                const double* __restrict__ diagR, const double* __restrict__ innd,
                                                                const double* __restrict__ Rmeas, double* __restrict__ P,
                                                                double* __restrict__ err, double* __restrict__ HP,
                                                                double* __restrict__ Kt, double* __restrict__ H_dense, int Mmax,
                                                                const EditOp* __restrict__ ops, const int* __restrict__ ops_first,
                                                                const int* __restrict__ nops, uint32_t* __restrict__ kt32,
                                                                uint32_t* __restrict__ hp32, int Npad, int KCmax, int full_j) {
  extern __shared__ __align__(16) double sm[];
  const int b = blockIdx.x, tid = threadIdx.x;
  const int M = SPARSE ? 2 * nsel[b] : Mdense;
  if (ops) apply_edits(N, P + (size_t)b * N * N, ops + ops_first[b], nops[b], tid, GAIN_THREADS);  // the post-gate edit list (uniform over the CTA)
  const double* Pb = P + (size_t)b * N * N;  // (no __restrict__: the edits above wrote P, the loads below must not take the non-coherent path)
  double* __restrict__ HPb = HP + (size_t)b * Mmax * N;
  double* __restrict__ Ktb = Kt + (size_t)b * Mmax * N;
  double* __restrict__ errb = err + (size_t)b * N;
  if (M == 0) {
    for (int j = tid; j < N; j += GAIN_THREADS) errb[j] = 0.0;
    return;
  }
  // shared: S (M x M), inn (M), [sparse] Hval (M x 21), Hcol (M x 21 ints)
  double* S = sm;
  double* inn = S + (size_t)Mmax * Mmax;
  double* Hval = inn + Mmax;
  int* Hcol = reinterpret_cast<int*>(Hval + (size_t)(SPARSE ? Mmax * kHnnz : 0));
  __shared__ int bad;
  if (tid == 0) bad = 0;

  if (SPARSE) {
    for (int t = tid; t < M * kHnnz; t += GAIN_THREADS) {
      const int r = t / kHnnz, k = t - r * kHnnz;
      const FeatJac& f = jac[(size_t)b * lay.F + sel[(size_t)b * lay.F + (r >> 1)]];
      // FillJacobianBlock: H(:, goff:goff+3) <- J(:, goff+3:goff+6); H(:, goff+3:goff+6) stays 0
      // full_j: the rows of J() as they are (OnePointRANSAC's low-innovation update, update.cpp:318-330)
      double v = f.J[r & 1][k];
      if (!full_j) {
        if (k >= 12 && k < 15) v = f.J[r & 1][k + 3];
        else if (k >= 15 && k < 18) v = 0.0;
      }
      Hval[t] = v;
      Hcol[t] = jac_col(k, f.goff, f.foff);
      if (k == 0) inn[r] = f.inn[r & 1];
    }
  } else {
    for (int r = tid; r < M; r += GAIN_THREADS) inn[r] = innd[(size_t)b * M + r];
  }
  __syncthreads();
  if (SPARSE && H_dense) {
    double* __restrict__ Hb = H_dense + (size_t)b * Mmax * N;
    for (int t = tid; t < M * N; t += GAIN_THREADS) Hb[t] = 0.0;
    __syncthreads();
    for (int t = tid; t < M * kHnnz; t += GAIN_THREADS) Hb[(size_t)(t / kHnnz) * N + Hcol[t]] = Hval[t];
  }
  // ---- a. HP = H P
  for (int t = tid; t < M * N; t += GAIN_THREADS) {
    const int r = t / N, j = t - r * N;
    double acc = 0.0;
    if (SPARSE) {
#pragma unroll
      for (int k = 0; k < kHnnz; ++k) acc += Hval[r * kHnnz + k] * Pb[(size_t)Hcol[r * kHnnz + k] * N + j];
    } else {
      const double* __restrict__ hr = Hd + ((size_t)b * M + r) * N;
      for (int k = 0; k < N; ++k) acc += hr[k] * Pb[(size_t)k * N + j];
    }
    HPb[t] = acc;
  }
  __syncthreads();
  // ---- b. S = HP H^T + R (lower triangle incl. diagonal is what Cholesky reads; fill both)
  for (int t = tid; t < M * M; t += GAIN_THREADS) {
    const int r = t / M, s = t - r * M;
    double acc = 0.0;
    if (SPARSE) {
#pragma unroll
      for (int k = 0; k < kHnnz; ++k) acc += HPb[(size_t)r * N + Hcol[s * kHnnz + k]] * Hval[s * kHnnz + k];
      if (r == s) acc += Rmeas[b];
    } else {
      const double* __restrict__ hs = Hd + ((size_t)b * M + s) * N;
      for (int k = 0; k < N; ++k) acc += HPb[(size_t)r * N + k] * hs[k];
      if (r == s) acc += diagR[(size_t)b * M + r];
    }
    S[r * Mmax + s] = acc;
  }
  __syncthreads();
  // ---- c. Cholesky S = L L^T (right-looking, in place in the lower triangle)
  for (int k = 0; k < M; ++k) {
    if (tid == 0) {
      const double dkk = S[k * Mmax + k];
      if (!(dkk > 0.0)) bad = 1;
      S[k * Mmax + k] = sqrt(dkk);
    }
    __syncthreads();
    const double inv = 1.0 / S[k * Mmax + k];
    for (int i = k + 1 + tid; i < M; i += GAIN_THREADS) S[i * Mmax + k] *= inv;
    __syncthreads();
    const int rem = M - k - 1;
    for (int t = tid; t < rem * rem; t += GAIN_THREADS) {
      const int ii = t / rem, jj = t - ii * rem;
      if (jj <= ii) {
        const int i = k + 1 + ii, j = k + 1 + jj;
        S[i * Mmax + j] -= S[i * Mmax + k] * S[j * Mmax + k];
      }
    }
    __syncthreads();
  }
  // ---- d. K^T = S^-1 HP by forward/back substitution, one thread per state column; err = K inn
  for (int j = tid; j < N; j += GAIN_THREADS) {
    for (int r = 0; r < M; ++r) {
      double acc = HPb[(size_t)r * N + j];
      for (int t = 0; t < r; ++t) acc -= S[r * Mmax + t] * Ktb[(size_t)t * N + j];
      Ktb[(size_t)r * N + j] = acc / S[r * Mmax + r];
    }
    double e = 0.0;
    for (int r = M - 1; r >= 0; --r) {
      double acc = Ktb[(size_t)r * N + j];
      for (int t = r + 1; t < M; ++t) acc -= S[t * Mmax + r] * Ktb[(size_t)t * N + j];
      acc /= S[r * Mmax + r];
      Ktb[(size_t)r * N + j] = acc;
      e += acc * inn[r];
    }
    if (bad) {  // S not positive definite: publish NaN err and a zero gain, so that the covariance downdate that follows is a no-op
      for (int r = 0; r < M; ++r) Ktb[(size_t)r * N + j] = 0.0;
      e = nan("");
    }
    errb[j] = e;
  }
  // ---- e. (tensor-core downdate only) K^T and HP once more as TF32 hi / lo words in the layout ekf_cov_tc2_kernel's TMA boxes expect:
  // [filter][hi|lo][k / 4][state column][4].  Thread j converts its own column (the values it has just written), 16-byte stores that
  // are contiguous across the threads; columns N .. Npad and rows M .. 32 * ceil(M / 32) are zero.
  if (kt32) {
    const int kchunks = ((M + 31) / 32) * 8;
    const size_t slab = (size_t)KCmax * Npad * 4;  // words of one (filter, hi|lo) slab
    uint32_t* __restrict__ kH = kt32 + (size_t)b * 2 * slab;
    uint32_t* __restrict__ hH = hp32 + (size_t)b * 2 * slab;
    for (int j = tid; j < Npad; j += GAIN_THREADS) {
      for (int kc = 0; kc < kchunks; ++kc) {
        uint4 kh = make_uint4(0, 0, 0, 0), kl = kh, hh = kh, hl = kh;
        if (j < N) {
          uint32_t* khp = &kh.x; uint32_t* klp = &kl.x; uint32_t* hhp = &hh.x; uint32_t* hlp = &hl.x;
#pragma unroll
          for (int q = 0; q < 4; ++q) {
            const int r = 4 * kc + q;
            if (r < M) {
              const double kv = Ktb[(size_t)r * N + j], hv = HPb[(size_t)r * N + j];
              uint32_t t;
              asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(t) : "f"((float)kv));
              khp[q] = t;
              asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(klp[q]) : "f"((float)(kv - (double)__uint_as_float(t))));
              asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(t) : "f"((float)hv));
              hhp[q] = t;
              asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(hlp[q]) : "f"((float)(hv - (double)__uint_as_float(t))));
            }
          }
        }
        const size_t o = ((size_t)kc * Npad + j) * 4;
        *reinterpret_cast<uint4*>(kH + o) = kh;
        *reinterpret_cast<uint4*>(kH + slab + o) = kl;
        *reinterpret_cast<uint4*>(hH + o) = hh;
        *reinterpret_cast<uint4*>(hH + slab + o) = hl;
      }
    }
  }
}

constexpr int CT = 32;  // covariance tile
__global__ void __launch_bounds__(256) ekf_cov_kernel(int N, const int* __restrict__ nsel, int Mdense, int Mmax,
                                                      const double* __restrict__ HP, const double* __restrict__ Kt,
                                                      double* __restrict__ P) {
  const int b = blockIdx.z;
  const int M = nsel ? 2 * nsel[b] : Mdense;
  const int ti = blockIdx.y, tj = blockIdx.x;
  if (M == 0 || ti > tj) return;
  __shared__ double sK[16][CT + 1], sH[16][CT + 1];
  const double* __restrict__ HPb = HP + (size_t)b * Mmax * N;
  const double* __restrict__ Ktb = Kt + (size_t)b * Mmax * N;
  double* __restrict__ Pb = P + (size_t)b * N * N;
  const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;  // 16 x 16 threads, 2 x 2 outputs each
  const int i0 = ti * CT, j0 = tj * CT;
  double acc[2][2] = {{0, 0}, {0, 0}};
  for (int r0 = 0; r0 < M; r0 += 16) {
    for (int t = threadIdx.x; t < 16 * CT; t += 256) {
      const int rr = t / CT, c = t - rr * CT;
      const int r = r0 + rr;
      sK[rr][c] = (r < M && i0 + c < N) ? Ktb[(size_t)r * N + i0 + c] : 0.0;
      sH[rr][c] = (r < M && j0 + c < N) ? HPb[(size_t)r * N + j0 + c] : 0.0;
    }
    __syncthreads();
#pragma unroll
    for (int rr = 0; rr < 16; ++rr) {
      const double k0 = sK[rr][ty], k1 = sK[rr][ty + 16], h0 = sH[rr][tx], h1 = sH[rr][tx + 16];
      acc[0][0] += k0 * h0;
      acc[0][1] += k0 * h1;
      acc[1][0] += k1 * h0;
      acc[1][1] += k1 * h1;
    }
    __syncthreads();
  }
#pragma unroll
  for (int a = 0; a < 2; ++a)
#pragma unroll
    for (int c = 0; c < 2; ++c) {
      const int i = i0 + ty + 16 * a, j = j0 + tx + 16 * c;
      if (i < N && j < N && i <= j) {
        const double v = Pb[(size_t)i * N + j] - acc[a][c];
        Pb[(size_t)i * N + j] = v;
        if (i != j) Pb[(size_t)j * N + i] = v;
      }
    }
}

static size_t gain_smem(int Mmax, bool sparse) {
  size_t s = sizeof(double) * ((size_t)Mmax * Mmax + Mmax);
  if (sparse) s += (size_t)Mmax * kHnnz * (sizeof(double) + sizeof(int));
  return s;
}

int ekf_gain_max_rows(bool sparse) {
  int m = 0;
  while (gain_smem(m + 1, sparse) <= kSmemOptin) ++m;
  return m;
}

int launch_ekf_update(cudaStream_t st, EkfLayout lay, const FeatJac* jac, const int* sel, const int* nsel, const double* Rmeas,
                      double* P, double* err, double* HP, double* Kt, double* H_dense, int batch, int tensor_core, const EditOp* ops,
                      const int* ops_first, const int* nops, const TcOperands* tc, int full_j) {
  const int N = lay.N(), Mmax = 2 * lay.F;
  XB_REQUIRE(Mmax <= ekf_gain_max_rows(true), "EKF update: 2*F too large for the shared-memory Cholesky");
  const bool tc2 = tensor_core && tc && tc->kt32;
  if (tc2) XB_REQUIRE(Mmax <= ekf_cov_tc2_max_rows(), "EKF update: 2*F too large for the tensor-core downdate's resident A operand");
  const size_t smem = gain_smem(Mmax, true);
  {  // one attribute call per size, not one per launch (every CUDA call of a driver thread contends with the other batches' drivers)
    static std::atomic<size_t> attr{0};
    if (smem > attr.load(std::memory_order_relaxed)) {
      XB_CUDA(cudaFuncSetAttribute(ekf_gain_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
      attr.store(smem, std::memory_order_relaxed);
    }
  }
  ProfRec* pi_ = Prof::get().start("ekf_gain", st);
  ekf_gain_kernel<true><<<batch, GAIN_THREADS, smem, st>>>(N, lay, jac, sel, nsel, 0, nullptr, nullptr, nullptr, Rmeas, P, err, HP,
                                                          Kt, H_dense, Mmax, ops, ops_first, nops, tc2 ? tc->kt32 : nullptr, tc2 ? tc->hp32 : nullptr,
                                                          tc2 ? tc->Npad : 0, tc2 ? tc->KCmax : 0, full_j);
  Prof::get().stop(pi_, st);
  if (tc2) return launch_ekf_cov_tc2(st, N, nsel, 0, *tc, P, batch);
  if (tensor_core) return launch_ekf_cov_tc(st, N, nsel, 0, Mmax, HP, Kt, P, batch);
  const int nt = (N + CT - 1) / CT;
  {
    ProfScope ps("ekf_cov", st);
    ekf_cov_kernel<<<dim3(nt, nt, batch), 256, 0, st>>>(N, nsel, 0, Mmax, HP, Kt, P);
  }
  XB_CUDA(cudaGetLastError());
  return 0;
}

int launch_ekf_update_dense(cudaStream_t st, int N, int M, const double* H, const double* diagR, const double* inn, double* P,
                            double* err, double* HP, double* Kt, int batch, int tensor_core, const TcOperands* tc) {
  XB_REQUIRE(M <= ekf_gain_max_rows(false), "EKF update: M too large for the shared-memory Cholesky");
  const bool tc2 = tensor_core && tc && tc->kt32;
  if (tc2) XB_REQUIRE(M <= ekf_cov_tc2_max_rows(), "EKF update: M too large for the tensor-core downdate's resident A operand");
  const size_t smem = gain_smem(M, false);
  XB_CUDA(cudaFuncSetAttribute(ekf_gain_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  EkfLayout lay{0, 0};
  {
    ProfScope pg("ekf_gain", st);
    ekf_gain_kernel<false><<<batch, GAIN_THREADS, smem, st>>>(N, lay, nullptr, nullptr, nullptr, M, H, diagR, inn, nullptr, P, err,
                                                             HP, Kt, nullptr, M, nullptr, nullptr, nullptr, tc2 ? tc->kt32 : nullptr,
                                                             tc2 ? tc->hp32 : nullptr, tc2 ? tc->Npad : 0, tc2 ? tc->KCmax : 0, 0);
  }
  if (tc2) return launch_ekf_cov_tc2(st, N, nullptr, M, *tc, P, batch);
  if (tensor_core) return launch_ekf_cov_tc(st, N, nullptr, M, M, HP, Kt, P, batch);
  const int nt = (N + CT - 1) / CT;
  {
    ProfScope pc("ekf_cov", st);
    ekf_cov_kernel<<<dim3(nt, nt, batch), 256, 0, st>>>(N, nullptr, M, M, HP, Kt, P);
  }
  XB_CUDA(cudaGetLastError());
  return 0;
}

// ------------------------------------------------------------------------------------------
// Covariance edit list: the reference edits P in many tiny steps per frame
// (/root/reference/src/estimator.cpp:739-846, :1362-1391, :1474-1478); with P device-resident
// the host queues them and one launch applies them in order.
// ------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) cov_edit_kernel(int N, double* __restrict__ P, const EditOp* __restrict__ ops,
                                                       const int* __restrict__ nops, int max_ops, const int* __restrict__ first) {
  const int b = blockIdx.x;
  apply_edits(N, P + (size_t)b * N * N, ops + (first ? (size_t)first[b] : (size_t)b * max_ops), nops[b], threadIdx.x, 256);
}

// first (device, optional): start of filter b's list inside a packed ops array; null = filter b owns ops[b * max_ops ...)
int launch_cov_edit(cudaStream_t st, int N, double* P, const EditOp* ops, const int* nops, int max_ops, int batch, const int* first) {
  ProfScope ps("cov_edit", st);
  cov_edit_kernel<<<batch, 256, 0, st>>>(N, P, ops, nops, max_ops, first);
  XB_CUDA(cudaGetLastError());
  return 0;
}

// ------------------------------------------------------------------------------------------
// Propagation strips (/root/reference/src/princedormand.cpp:208-215, rk4.cpp:95-102, composed over
// the sub-steps of all IMU samples since the previous frame): the 23x23 motion block is
// integrated on the host in fp64; the device applies Phi to the motion/structure strips.
// ------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) cov_propagate_kernel(int N, double* __restrict__ P, const double* __restrict__ Phi,
                                                            const double* __restrict__ Pmm, const unsigned char* __restrict__ active) {
  const int b = blockIdx.x, tid = threadIdx.x;
  if (active && !active[b]) return;
  __shared__ double sPhi[23 * 23];
  double* __restrict__ Pb = P + (size_t)b * N * N;
  for (int t = tid; t < 23 * 23; t += 256) sPhi[t] = Phi[(size_t)b * 529 + t];
  __syncthreads();
  for (int j = 23 + tid; j < N; j += 256) {
    double col[23];
#pragma unroll
    for (int k = 0; k < 23; ++k) col[k] = Pb[(size_t)k * N + j];
#pragma unroll 1
    for (int i = 0; i < 23; ++i) {
      double acc = 0.0;
#pragma unroll
      for (int k = 0; k < 23; ++k) acc += sPhi[i * 23 + k] * col[k];
      Pb[(size_t)i * N + j] = acc;
      Pb[(size_t)j * N + i] = acc;
    }
  }
  for (int t = tid; t < 529; t += 256) Pb[(size_t)(t / 23) * N + t % 23] = Pmm[(size_t)b * 529 + t];
}

int launch_cov_propagate(cudaStream_t st, int N, double* P, const double* Phi, const double* Pmm, const unsigned char* active,
                         int batch) {
  ProfScope ps("cov_propagate", st);
  cov_propagate_kernel<<<batch, 256, 0, st>>>(N, P, Phi, Pmm, active);
  XB_CUDA(cudaGetLastError());
  return 0;
}

// Pack what the host needs after an update into one contiguous block per filter:
// [err (N) | P[0:23,0:23] (529) | diag(P) (N)]  -> a single D2H copy per batch.
__global__ void __launch_bounds__(256) pack_state_kernel(int N, const double* __restrict__ P, const double* __restrict__ err,
                                                         double* __restrict__ out) {
  const int b = blockIdx.x, tid = threadIdx.x;
  const double* __restrict__ Pb = P + (size_t)b * N * N;
  double* __restrict__ ob = out + (size_t)b * (2 * N + 529);
  for (int t = tid; t < N; t += 256) {
    ob[t] = err[(size_t)b * N + t];
    ob[N + 529 + t] = Pb[(size_t)t * N + t];
  }
  for (int t = tid; t < 529; t += 256) ob[N + t] = Pb[(size_t)(t / 23) * N + t % 23];
}
int launch_pack_state(cudaStream_t st, int N, const double* P, const double* err, double* out, int batch) {
  ProfScope ps("pack_state", st);
  pack_state_kernel<<<batch, 256, 0, st>>>(N, P, err, out);
  XB_CUDA(cudaGetLastError());
  return 0;
}

// Initial covariance of filters first .. first + count - 1 (Estimator::Estimator, estimator.cpp:258-302): identity with the filter's own
// 23 x 23 motion block.  Grid: (column tiles, count); thread = one column of one row chunk, so the stores of a warp are contiguous.
__global__ void __launch_bounds__(256) cov_init_kernel(int N, double* __restrict__ P, const double* __restrict__ Pmm, int first) {
  const int b = first + blockIdx.y;
  const int j = blockIdx.x * 256 + threadIdx.x;
  if (j >= N) return;
  double* __restrict__ Pb = P + (size_t)b * N * N;
  const double* __restrict__ Mb = Pmm + (size_t)b * 529;
  for (int i = 0; i < N; ++i) Pb[(size_t)i * N + j] = (i < 23 && j < 23) ? Mb[i * 23 + j] : (i == j ? 1.0 : 0.0);
}
int launch_cov_init(cudaStream_t st, int N, double* P, const double* Pmm, int first, int count) {
  if (count <= 0) return 0;
  ProfScope ps("cov_init", st);
  cov_init_kernel<<<dim3((N + 255) / 256, count), 256, 0, st>>>(N, P, Pmm, first);
  XB_CUDA(cudaGetLastError());
  return 0;
}

// ------------------------------------------------------------------------------------------
// IMU covariance propagation: the covariance side of Estimator::Propagate -> PrinceDormand / RK4
// (/root/reference/src/estimator.cpp:539-704, src/princedormand.cpp:85-221, src/rk4.cpp:35-103).
// One block per filter consumes the per-sub-step records the host wrote while integrating the nominal
// state (kernels.h: ImuStep) and rebuilds what every Runge-Kutta stage needs from them.  Structure
// used: only the Wsb/Tsb/Vsb rows of F are non-zero, so F*X is a 9 x 23 strip and  Pdot = [A;0] + [A;0]^T + G Q G^T,  A = F[0:9,:] P,  G Q G^T block diagonal
// (Q diagonal).  At the end the motion/structure strips get Phi = prod(I + FK h) (rows >= 9 = identity).
// ------------------------------------------------------------------------------------------
struct F9s {  // shared-memory image of the non-zero blocks of F and of R (+ the stage's calibrated rates)
  double dW[9], dVW[9], dVba[9], dVg[6], R[9], gc[3], ac[3];
};
// element (i, j), i < 9, of F[0:9,:] * B for a 23-column B; lt9: rows >= 9 of B are zero
__device__ __forceinline__ double f9_elem(const F9s& f, const double* B, int i, int j, bool lt9) {
  const int blk = i / 3, r = i - 3 * blk;
  if (blk == 0) {
    double v = f.dW[3 * r] * B[j] + f.dW[3 * r + 1] * B[23 + j] + f.dW[3 * r + 2] * B[46 + j];
    if (!lt9) v -= B[(9 + r) * 23 + j];
    return v;
  }
  if (blk == 1) return B[(6 + r) * 23 + j];
  double v = f.dVW[3 * r] * B[j] + f.dVW[3 * r + 1] * B[23 + j] + f.dVW[3 * r + 2] * B[46 + j];
  if (!lt9)
    v += f.dVba[3 * r] * B[12 * 23 + j] + f.dVba[3 * r + 1] * B[13 * 23 + j] + f.dVba[3 * r + 2] * B[14 * 23 + j] +
         f.dVg[2 * r] * B[21 * 23 + j] + f.dVg[2 * r + 1] * B[22 * 23 + j];
  return v;
}
__device__ __forceinline__ double f9_dense(const F9s& f, int i, int j) {  // F[i][j], i < 9
  const int blk = i / 3, r = i - 3 * blk;
  if (blk == 0) return j < 3 ? f.dW[3 * r + j] : (j == 9 + r ? -1.0 : 0.0);
  if (blk == 1) return j == 6 + r ? 1.0 : 0.0;
  if (j < 3) return f.dVW[3 * r + j];
  if (j >= 12 && j < 15) return f.dVba[3 * r + j - 12];
  if (j >= 21) return f.dVg[2 * r + j - 21];
  return 0.0;
}
__device__ __forceinline__ double hat_elem(const double* w, int k, int j) {  // hat(w)[k][j]
  if (k == j) return 0.0;
  const int o = 3 - k - j;  // the remaining index
  const double sgn = ((j - k + 3) % 3 == 1) ? -1.0 : 1.0;  // hat: [0,-w2,w1; w2,0,-w0; -w1,w0,0]
  return sgn * w[o];
}

__constant__ double kApd[6][6] = {{2.0 / 9, 0, 0, 0, 0, 0},
                                  {1.0 / 12, 3.0 / 12, 0, 0, 0, 0},
                                  {55.0 / 324, -75.0 / 324, 200.0 / 324, 0, 0, 0},
                                  {83.0 / 330, -195.0 / 330, 305.0 / 330, 27.0 / 330, 0, 0},
                                  {-19.0 / 28, 63.0 / 28, 4.0 / 28, -108.0 / 28, 88.0 / 28, 0},
                                  {38.0 / 400, 0, 240.0 / 400, -243.0 / 400, 330.0 / 400, 35.0 / 400}};
__constant__ double kBpd[7] = {0.0862, 0.0, 0.6660, -0.7857, 0.9570, 0.0965, -0.0200};
__constant__ double kArk[3][6] = {{0.5, 0, 0, 0, 0, 0}, {0, 0.5, 0, 0, 0, 0}, {0, 0, 1.0, 0, 0, 0}};
__constant__ double kBrk[4] = {1.0 / 6, 2.0 / 6, 2.0 / 6, 1.0 / 6};

constexpr int IMU_THREADS = 256;
constexpr int IMU_CHUNK = 56;
// Stage images of the n stages [c0, c0 + n) of a filter (c0, n: whole sub-steps of nst stages) from its sub-step records.
// Pass 1, one thread per stage: the stage's rotation and rates (imu_stage_from_step).  Pass 2, nine threads per stage: the
// non-zero blocks of F,  dW = -hat(gc), dVW = -R hat(ac), dVba = -R, dVg = (-R hat(g))[:, :2].  sH[q] = the h of stage q's sub-step.
__device__ __forceinline__ void imu_load_chunk(const ImuStep* __restrict__ stp, int c0, int n, int nst, const ImuConst& c, F9s* sFc, double* sH,
                                               int tid) {
  const bool pd = nst == 7;
  for (int u = tid; u < n; u += IMU_THREADS) {
    const int k = (c0 + u) / nst, s = (c0 + u) - nst * k;
    F9s& f = sFc[u];
    M3 R;
    V3 gc, ac;
    imu_stage_from_step(stp[k], s, pd, &R, &gc, &ac);
#pragma unroll
    for (int e = 0; e < 9; ++e) f.R[e] = R.m[e];
#pragma unroll
    for (int e = 0; e < 3; ++e) { f.gc[e] = gc.v[e]; f.ac[e] = ac.v[e]; }
    sH[u] = stp[k].h;
  }
  __syncthreads();
  for (int u = tid; u < n * 9; u += IMU_THREADS) {
    const int q = u / 9, e = u - 9 * q;
    const int i = e / 3, j = e - 3 * i;
    F9s& f = sFc[q];
    const double* Rm = f.R;
    f.dVba[e] = -Rm[e];
    f.dW[e] = -hat_elem(f.gc, i, j);
    double v = 0, vg = 0;
    for (int k = 0; k < 3; ++k) {
      v += Rm[3 * i + k] * hat_elem(f.ac, k, j);
      vg += Rm[3 * i + k] * hat_elem(c.g, k, j);
    }
    f.dVW[e] = -v;
    if (j < 2) f.dVg[2 * i + j] = -vg;
  }
}

__device__ __forceinline__ double v_block(const F9s& f, const ImuConst& c, int e) {  // (R diag(qa) R^T)[e / 3][e % 3]
  const int i = e / 3, j = e - 3 * i;
  return f.R[3 * i] * c.qimu[3] * f.R[3 * j] + f.R[3 * i + 1] * c.qimu[4] * f.R[3 * j + 1] + f.R[3 * i + 2] * c.qimu[5] * f.R[3 * j + 2];
}

// Covariance propagation over a filter's queued IMU sub-steps, one CTA per filter: the Runge-Kutta (Prince-Dormand or RK4) stage
// chain of the 23 x 23 motion block, the 9 x 23 strips of Phi = prod (I + FK h), and at the end rows 0..8 of P against the feature
// columns (P[0:9, 23:N] = Phi P[0:23, 23:N]).  Every thread owns fixed elements: a strip thread keeps its FK[q] / A[q] of all stages
// of the sub-step in registers, a P thread keeps its covariance entries in registers.  So the Runge-Kutta combinations need no
// shared-memory round trip and no index tables, and the stage chain has two barriers per stage (double-buffered Acc / SA / CV).
// (A formulation with shared-memory index tables and three barriers per stage spends its issue slots on index arithmetic and its
// stalls at barriers rather than on DFMA, and takes 2.2 times as long: DESIGN.md section 4.)
__global__ void __launch_bounds__(IMU_THREADS) imu_cov_propagate_kernel(int N, double* __restrict__ P, const ImuStep* __restrict__ steps,
                                                                        const int* __restrict__ first, const int* __restrict__ nsteps,
                                                                        const ImuConst* __restrict__ cst) {
  const int b = blockIdx.x, tid = threadIdx.x;
  if (nsteps[b] == 0) return;
  __shared__ double sP[529], sP0[529], sAcc[2][207], sSA[2][207], sPhi[2][207], sCV[2][9], sGc[23];
  __shared__ ImuConst c;
  if (tid < (int)(sizeof(ImuConst) / 8)) reinterpret_cast<double*>(&c)[tid] = reinterpret_cast<const double*>(cst + b)[tid];
  double* __restrict__ Pb = P + (size_t)b * N * N;
  const ImuStep* __restrict__ stp = steps + first[b];
  // ---- fixed ownership
  const bool strip = tid < 207;               // element (si, sj) of the 9 x 23 strips
  const int si = strip ? tid / 23 : 0, sj = strip ? tid - 23 * si : 0;
  const bool vthr = tid >= 224 && tid < 233;  // element ve of the 3 x 3 accel-noise block (its own warp)
  const int ve = vthr ? tid - 224 : 0;
  int pi[3], pj[3];                           // covariance entries tid, tid + 256, tid + 512
  bool pv[3];
  double preg[3];
#pragma unroll
  for (int m = 0; m < 3; ++m) {
    const int t = tid + IMU_THREADS * m;
    pv[m] = t < 529;
    pi[m] = pv[m] ? t / 23 : 0;
    pj[m] = pv[m] ? t - 23 * pi[m] : 0;
    preg[m] = pv[m] ? Pb[(size_t)pi[m] * N + pj[m]] : 0.0;
    if (pv[m]) sP[t] = preg[m];
  }
  if (strip) sPhi[0][tid] = si == sj ? 1.0 : 0.0;
  __syncthreads();
  const int nst = c.stages_per_step;
  const int nall = nsteps[b] * nst;  // stages
  const bool pd = nst == 7;
  if (tid < 23) {  // state-independent diagonal of G Q G^T
    double v = 0.0;
    if (tid < 3) v = c.qimu[tid];
    else if (tid >= 9 && tid < 12) v = c.qimu[6 + tid - 9];
    else if (tid >= 12 && tid < 15) v = c.qimu[9 + tid - 12];
    sGc[tid] = v;
  }
  // Stages are consumed in chunks of IMU_CHUNK (a multiple of both 7 and 4 stages per substep): the non-zero
  // blocks of F of every stage of the chunk are built in parallel up front (imu_load_chunk), so the serial stage chain below
  // never waits on global memory or on the stage rotations.
  extern __shared__ __align__(16) unsigned char imu_dyn[];
  F9s* sFc = reinterpret_cast<F9s*>(imu_dyn);
  double* sH = reinterpret_cast<double*>(sFc + IMU_CHUNK);
  auto load_chunk = [&](int c0) {
    __syncthreads();  // the previous chunk is no longer read
    imu_load_chunk(stp, c0, min(IMU_CHUNK, nall - c0), nst, c, sFc, sH, tid);
    __syncthreads();
  };
  // increment of covariance entry (i, j): strip_sym(SA) + sw * diag(GQG const) + CV on the velocity block
  auto p_inc = [&](int i, int j, int buf, double sw) {
    double inc = (i < 9 ? sSA[buf][i * 23 + j] : 0.0) + (j < 9 ? sSA[buf][j * 23 + i] : 0.0);
    if (i == j) inc += sw * sGc[i];
    if (i >= 6 && i < 9 && j >= 6 && j < 9) inc += sCV[buf][(i - 6) * 3 + j - 6];
    return inc;
  };
  int buf = 0, pb = 0;
  for (int base = 0; base + nst <= nall; base += nst) {
    if (base % IMU_CHUNK == 0) load_chunk(base);
    const int cb = base % IMU_CHUNK;
    const double henc = sH[cb];
    const double h = fabs(henc);
    double FK[7], A[7], V[7];
#pragma unroll
    for (int q = 0; q < 7; ++q) FK[q] = A[q] = V[q] = 0.0;
    {
      const F9s& f = sFc[cb];
      if (strip) {
        FK[0] = f9_dense(f, si, sj);
        A[0] = f9_elem(f, sP, si, sj, false);
      }
      if (vthr) V[0] = v_block(f, c, ve);
    }
#pragma unroll
    for (int s = 1; s < 7; ++s) {
      if (s < nst) {
        const double* a = pd ? kApd[s - 1] : kArk[s - 1];
        double sa = 0;
#pragma unroll
        for (int q = 0; q < s; ++q) sa += a[q];
        if (strip) {
          double f = 0, p = 0;
#pragma unroll
          for (int q = 0; q < s; ++q) { f += a[q] * FK[q]; p += a[q] * A[q]; }
          sAcc[buf][tid] = f;
          sSA[buf][tid] = p;
        }
        if (vthr) {
          double v = 0;
#pragma unroll
          for (int q = 0; q < s; ++q) v += a[q] * V[q];
          sCV[buf][ve] = v;
        }
        __syncthreads();
#pragma unroll
        for (int m = 0; m < 3; ++m)
          if (pv[m]) sP0[tid + IMU_THREADS * m] = preg[m] + p_inc(pi[m], pj[m], buf, sa) * h;
        __syncthreads();
        const F9s& f = sFc[cb + s];
        if (strip) {
          const double fd = f9_dense(f, si, sj);
          FK[s] = fd + f9_elem(f, sAcc[buf], si, sj, true) * h;
          A[s] = f9_elem(f, sP0, si, sj, false);
        }
        if (vthr) V[s] = v_block(f, c, ve);
        buf ^= 1;
      }
    }
    const double* bw = pd ? kBpd : kBrk;
    double sb = 0;
#pragma unroll
    for (int q = 0; q < 7; ++q)
      if (q < nst) sb += bw[q];
    if (strip) {
      double f = 0, p = 0;
#pragma unroll
      for (int q = 0; q < 7; ++q)
        if (q < nst) { f += bw[q] * FK[q]; p += bw[q] * A[q]; }
      sAcc[buf][tid] = ((si == sj) ? 1.0 : 0.0) + f * h;  // rows 0..8 of I + FK h
      sSA[buf][tid] = p;
    }
    if (vthr) {
      double v = 0;
#pragma unroll
      for (int q = 0; q < 7; ++q)
        if (q < nst) v += bw[q] * V[q];
      sCV[buf][ve] = v;
    }
    __syncthreads();
#pragma unroll
    for (int m = 0; m < 3; ++m)
      if (pv[m]) {
        double v = preg[m] + p_inc(pi[m], pj[m], buf, sb) * h;
        if (henc < 0 && pi[m] == pj[m]) v += c.qmodel[pi[m]];  // end of a Propagate call: += Qmodel (diagonal)
        preg[m] = v;
        sP[tid + IMU_THREADS * m] = v;
      }
    if (strip) {  // Phi <- (I + FK h) Phi; rows >= 9 of both factors are identity rows
      double v = sj >= 9 ? sAcc[buf][si * 23 + sj] : 0.0;
#pragma unroll
      for (int k = 0; k < 9; ++k) v += sAcc[buf][si * 23 + k] * sPhi[pb][k * 23 + sj];
      sPhi[pb ^ 1][tid] = v;
    }
    pb ^= 1;
    buf ^= 1;
    __syncthreads();
  }
  // write back: motion block and strips (rows 0..8 change)
#pragma unroll
  for (int m = 0; m < 3; ++m)
    if (pv[m]) Pb[(size_t)pi[m] * N + pj[m]] = preg[m];
  const double* __restrict__ phi = sPhi[pb];
  for (int j = 23 + tid; j < N; j += IMU_THREADS) {
    double col[23];
#pragma unroll
    for (int k = 0; k < 23; ++k) col[k] = Pb[(size_t)k * N + j];
#pragma unroll 1
    for (int i = 0; i < 9; ++i) {
      double acc = 0.0;
#pragma unroll
      for (int k = 0; k < 23; ++k) acc += phi[i * 23 + k] * col[k];
      Pb[(size_t)i * N + j] = acc;
      Pb[(size_t)j * N + i] = acc;
    }
  }
}

int launch_imu_cov_propagate(cudaStream_t st, int N, double* P, const ImuStep* steps, const int* first, const int* nsteps,
                             const ImuConst* cst, int batch) {
  ProfScope ps("imu_cov_propagate", st);
  const size_t dyn = IMU_CHUNK * (sizeof(F9s) + sizeof(double));
  static bool attr_set = false;
  if (!attr_set) {
    XB_CUDA(cudaFuncSetAttribute(imu_cov_propagate_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)dyn));
    attr_set = true;
  }
  imu_cov_propagate_kernel<<<batch, IMU_THREADS, dyn, st>>>(N, P, steps, first, nsteps, cst);
  XB_CUDA(cudaGetLastError());
  return 0;
}

// ------------------------------------------------------------------------------------------
// Depth sub-filter: Feature::SubfilterUpdate (/root/reference/src/feature.cpp:246-297).
// ------------------------------------------------------------------------------------------
__global__ void subfilter_kernel(const CameraParams* __restrict__ cam, const double* __restrict__ X,
                                 const SubfilterIn* __restrict__ in, SubfilterOut* __restrict__ out, int n, double Rtri,
                                 double mh_thresh) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const SubfilterIn f = in[i];
  const double* Xb = X + (size_t)f.filter * kPoseDoubles;
  M3 Rsb, Rbc, Rr;
  V3 Tsb, Tbc, Tr;
  for (int k = 0; k < 9; ++k) { Rsb.m[k] = Xb[k]; Rbc.m[k] = Xb[12 + k]; Rr.m[k] = f.ref[k]; }
  for (int k = 0; k < 3; ++k) { Tsb.v[k] = Xb[9 + k]; Tbc.v[k] = Xb[21 + k]; Tr.v[k] = f.ref[9 + k]; }
  const double z = exp(f.x[2]);
  const V3 Xc{{f.x[0] * z, f.x[1] * z, z}};
  const M3 dXc_dx{{z, 0, f.x[0] * z, 0, z, f.x[1] * z, 0, 0, z}};
  // gtot = (gsb gbc)^-1 (gref gbc)
  const M3 Rsc = m3_mul(Rsb, Rbc), Rrc = m3_mul(Rr, Rbc);
  const V3 Tsc = v3_add(m3_mulv(Rsb, Tbc), Tsb), Trc = v3_add(m3_mulv(Rr, Tbc), Tr);
  const M3 Rsc_t = m3_t(Rsc);
  const M3 Rtot = m3_mul(Rsc_t, Rrc);
  const V3 Ttot = m3_mulv(Rsc_t, v3_sub(Trc, Tsc));
  const V3 Xcn = v3_add(m3_mulv(Rtot, Xc), Ttot);
  const double iz = 1.0 / Xcn.v[2];
  const double P23[6] = {iz, 0, -Xcn.v[0] * iz * iz, 0, iz, -Xcn.v[1] * iz * iz};
  double u, v, Jc[4];
  camera_project(cam[f.filter], Xcn.v[0] * iz, Xcn.v[1] * iz, &u, &v, Jc);
  M23 d;
  for (int j = 0; j < 3; ++j) {
    d.m[j] = Jc[0] * P23[j] + Jc[1] * P23[3 + j];
    d.m[3 + j] = Jc[2] * P23[j] + Jc[3] * P23[3 + j];
  }
  const M23 H = m23_mul(m23_mul(d, Rtot), dXc_dx);
  const double r0 = f.xp[0] - u, r1 = f.xp[1] - v;
  // PHt (3x2), S = H P H^T + Rtri
  double PHt[6];
  for (int a = 0; a < 3; ++a)
    for (int c = 0; c < 2; ++c) PHt[2 * a + c] = f.P[3 * a] * H.m[3 * c] + f.P[3 * a + 1] * H.m[3 * c + 1] + f.P[3 * a + 2] * H.m[3 * c + 2];
  double S00 = H.m[0] * PHt[0] + H.m[1] * PHt[2] + H.m[2] * PHt[4] + Rtri;
  double S01 = H.m[0] * PHt[1] + H.m[1] * PHt[3] + H.m[2] * PHt[5];
  double S10 = H.m[3] * PHt[0] + H.m[4] * PHt[2] + H.m[5] * PHt[4];
  double S11 = H.m[3] * PHt[1] + H.m[4] * PHt[3] + H.m[5] * PHt[5] + Rtri;
  const double det0 = S00 * S11 - S01 * S10;
  const double ratio = (r0 * (S11 * r0 - S01 * r1) + r1 * (-S10 * r0 + S00 * r1)) / det0 / mh_thresh;
  double oc;
  if (ratio > 1) {
    S00 += Rtri * (ratio - 1);
    S11 += Rtri * (ratio - 1);
    oc = f.outlier_counter + sqrt(ratio);
  } else {
    oc = 0.0;
  }
  const double det = S00 * S11 - S01 * S10;
  const double Si[4] = {S11 / det, -S01 / det, -S10 / det, S00 / det};
  double K[6];  // 3x2 = PHt * Sinv
  for (int a = 0; a < 3; ++a) {
    K[2 * a] = PHt[2 * a] * Si[0] + PHt[2 * a + 1] * Si[2];
    K[2 * a + 1] = PHt[2 * a] * Si[1] + PHt[2 * a + 1] * Si[3];
  }
  SubfilterOut o;
  for (int a = 0; a < 3; ++a) o.x[a] = f.x[a] + K[2 * a] * r0 + K[2 * a + 1] * r1;
  double A[9];  // I - K H
  for (int a = 0; a < 3; ++a)
    for (int c = 0; c < 3; ++c) A[3 * a + c] = (a == c ? 1.0 : 0.0) - (K[2 * a] * H.m[c] + K[2 * a + 1] * H.m[3 + c]);
  double AP[9];
  for (int a = 0; a < 3; ++a)
    for (int c = 0; c < 3; ++c) AP[3 * a + c] = A[3 * a] * f.P[c] + A[3 * a + 1] * f.P[3 + c] + A[3 * a + 2] * f.P[6 + c];
  for (int a = 0; a < 3; ++a)
    for (int c = 0; c < 3; ++c)
      o.P[3 * a + c] = AP[3 * a] * A[3 * c] + AP[3 * a + 1] * A[3 * c + 1] + AP[3 * a + 2] * A[3 * c + 2] +
                       Rtri * (K[2 * a] * K[2 * c] + K[2 * a + 1] * K[2 * c + 1]);
  o.outlier_counter = oc;
  out[i] = o;
}

int launch_subfilter(cudaStream_t st, const CameraParams* cam, const double* X, const SubfilterIn* in, SubfilterOut* out, int n,
                     double Rtri, double mh_thresh) {
  if (n == 0) return 0;
  ProfScope ps("subfilter", st);
  subfilter_kernel<<<(n + 127) / 128, 128, 0, st>>>(cam, X, in, out, n, Rtri, mh_thresh);
  XB_CUDA(cudaGetLastError());
  return 0;
}

// ------------------------------------------------------------------------------------------
// OOS / MSCKF blocks + left-nullspace projection.
// Blocks: Feature::ComputeOOSJacobianInternal (/root/reference/src/oos.cpp:39-89).
// Projection: the reference multiplies by a basis of ker(Hf^T) from FullPivLU::kernel
// (/root/reference/src/helpers.cpp:13-23), which is neither unique nor orthonormal; we apply the
// three Householder reflectors that triangularise Hf and drop the first 3 rows, i.e. A = Q[:, 3:]
// is orthonormal (what the Givens variant, helpers.cpp:48-75, intends), so the projected noise
// stays Roos * I.  Parity is therefore on invariants (A^T Hf = 0, row space of A^T Hx).
// ------------------------------------------------------------------------------------------
constexpr int OOS_THREADS = 128;
constexpr int OOS_MAXROWS = 64;  // 2k <= 64

__global__ void __launch_bounds__(OOS_THREADS) oos_kernel(EkfLayout lay, const CameraParams* __restrict__ cam,
                                                          const double* __restrict__ gbc, const double* __restrict__ Xs,
                                                          const double* __restrict__ obs_pose, const int* __restrict__ obs_sind,
                                                          const double* __restrict__ obs_xp, int k, double* __restrict__ Hf,
                                                          double* __restrict__ Hx, double* __restrict__ inn,
                                                          double* __restrict__ Hx_proj, double* __restrict__ inn_proj) {
  const int f = blockIdx.x, tid = threadIdx.x;
  const int N = lay.N(), R2 = 2 * k;
  __shared__ double sHf[OOS_MAXROWS][3], sinn[OOS_MAXROWS], sv[OOS_MAXROWS];
  __shared__ double sbeta;
  double* __restrict__ Hxf = Hx + (size_t)f * R2 * N;
  for (int t = tid; t < R2 * N; t += OOS_THREADS) Hxf[t] = 0.0;
  __syncthreads();
  if (tid < k) {
    M3 Rbc, Rsb;
    V3 Tbc, Tsb;
    const double* gp = obs_pose + ((size_t)f * k + tid) * kGroupDoubles;
    for (int i = 0; i < 9; ++i) { Rbc.m[i] = gbc[i]; Rsb.m[i] = gp[i]; }
    for (int i = 0; i < 3; ++i) { Tbc.v[i] = gbc[9 + i]; Tsb.v[i] = gp[9 + i]; }
    const M3 Rsb_t = m3_t(Rsb), Rbc_t = m3_t(Rbc);
    const V3 X{{Xs[3 * f], Xs[3 * f + 1], Xs[3 * f + 2]}};
    const V3 Xb = m3_mulv(Rsb_t, v3_sub(X, Tsb));
    const V3 Xcn = m3_mulv(Rbc_t, v3_sub(Xb, Tbc));
    const double iz = 1.0 / Xcn.v[2];
    const double P23[6] = {iz, 0, -Xcn.v[0] * iz * iz, 0, iz, -Xcn.v[1] * iz * iz};
    double u, v, Jc[4];
    camera_project(cam[0], Xcn.v[0] * iz, Xcn.v[1] * iz, &u, &v, Jc);
    M23 d;
    for (int j = 0; j < 3; ++j) {
      d.m[j] = Jc[0] * P23[j] + Jc[1] * P23[3 + j];
      d.m[3 + j] = Jc[2] * P23[j] + Jc[3] * P23[3 + j];
    }
    const M23 dRbct = m23_mul(d, Rbc_t);
    const M23 hf = m23_mul(dRbct, Rsb_t);
    const M23 hW = m23_mul(dRbct, m3_hat(Xb));
    const M23 hT = m23_mul(dRbct, m3_neg(Rsb_t));
    const M23 hWbc = m23_mul(d, m3_hat(Xcn));
    const M23 hTbc = m23_mul(d, m3_neg(Rbc_t));
    const int goff = lay.goff(obs_sind[(size_t)f * k + tid]);
    for (int r = 0; r < 2; ++r) {
      const int row = 2 * tid + r;
      for (int j = 0; j < 3; ++j) {
        sHf[row][j] = hf.m[3 * r + j];
        Hxf[(size_t)row * N + goff + j] = hW.m[3 * r + j];
        Hxf[(size_t)row * N + goff + 3 + j] = hT.m[3 * r + j];
        Hxf[(size_t)row * N + 15 + j] = hWbc.m[3 * r + j];
        Hxf[(size_t)row * N + 18 + j] = hTbc.m[3 * r + j];
      }
      sinn[row] = obs_xp[((size_t)f * k + tid) * 2 + r] - (r == 0 ? u : v);
    }
  }
  __syncthreads();
  for (int t = tid; t < R2 * 3; t += OOS_THREADS) Hf[(size_t)f * R2 * 3 + t] = sHf[t / 3][t % 3];
  for (int t = tid; t < R2; t += OOS_THREADS) inn[(size_t)f * R2 + t] = sinn[t];
  // working copy of Hx for the projection
  double* __restrict__ W = Hx_proj ? Hx_proj + (size_t)f * R2 * N : nullptr;  // caller sizes Hx_proj as 2k x N scratch+output
  if (!W) return;
  for (int t = tid; t < R2 * N; t += OOS_THREADS) W[t] = Hxf[t];
  __syncthreads();
  for (int c = 0; c < 3; ++c) {
    if (tid == 0) {
      double nrm = 0.0;
      for (int r = c; r < R2; ++r) nrm += sHf[r][c] * sHf[r][c];
      nrm = sqrt(nrm);
      const double alpha = sHf[c][c] > 0 ? -nrm : nrm;
      double vnorm2 = 0.0;
      for (int r = c; r < R2; ++r) {
        sv[r] = sHf[r][c] - (r == c ? alpha : 0.0);
        vnorm2 += sv[r] * sv[r];
      }
      sbeta = vnorm2 > 0 ? 2.0 / vnorm2 : 0.0;
    }
    __syncthreads();
    // apply (I - beta v v^T) to Hf columns, inn (thread 0..3) and to the N columns of W
    if (tid < 4) {
      double dot = 0.0;
      for (int r = c; r < R2; ++r) dot += sv[r] * (tid < 3 ? sHf[r][tid] : sinn[r]);
      dot *= sbeta;
      for (int r = c; r < R2; ++r) {
        if (tid < 3) sHf[r][tid] -= dot * sv[r];
        else sinn[r] -= dot * sv[r];
      }
    }
    for (int j = tid; j < N; j += OOS_THREADS) {
      double dot = 0.0;
      for (int r = c; r < R2; ++r) dot += sv[r] * W[(size_t)r * N + j];
      dot *= sbeta;
      for (int r = c; r < R2; ++r) W[(size_t)r * N + j] -= dot * sv[r];
    }
    __syncthreads();
  }
  // rows 3.. are the projected system; compact them to the front of the output
  for (int r = 3; r < R2; ++r) {
    for (int j = tid; j < N; j += OOS_THREADS) W[(size_t)(r - 3) * N + j] = W[(size_t)r * N + j];
    __syncthreads();
  }
  for (int t = tid; t < R2 - 3; t += OOS_THREADS) inn_proj[(size_t)f * R2 + t] = sinn[t + 3];
}

int launch_oos(cudaStream_t st, EkfLayout lay, const CameraParams* cam, const double* Rbc_Tbc, const double* Xs,
               const double* obs_pose, const int* obs_sind, const double* obs_xp, int k, int nf, double* Hf, double* Hx,
               double* inn, double* Hx_proj, double* inn_proj) {
  XB_REQUIRE(2 * k <= OOS_MAXROWS && k >= 2, "OOS: 2 <= observations <= 32");
  if (nf == 0) return 0;
  oos_kernel<<<nf, OOS_THREADS, 0, st>>>(lay, cam, Rbc_Tbc, Xs, obs_pose, obs_sind, obs_xp, k, Hf, Hx, inn, Hx_proj, inn_proj);
  XB_CUDA(cudaGetLastError());
  return 0;
}

}  // namespace xb
