// Tensor-core form of the covariance downdate of the EKF measurement update.
//
// Reference: Estimator::UpdateJosephForm (src/estimator.cpp:1257-1288 of the reference).  After the gain
// kernel (ekf_kernels.cu) has produced HP = H P (M x N) and K^T = S^-1 HP (M x N), the only dense
// contraction left in the update is the rank-M downdate
//        P  <-  P - K (H P),      D[i][j] = sum_k Kt[k][i] * HP[k][j],   i, j < N, k < M.
// ekf_cov_kernel evaluates D in fp64 on the CUDA cores.  This file evaluates it on the Hopper tensor cores:
// wgmma.mma_async m64n32k8 .tf32 with fp32 accumulators in registers, operands split as
// x = hi + lo (both TF32) and D = Alo*Bhi + Ahi*Blo + Ahi*Bhi ("3xTF32": ~21 mantissa bits per product,
// fp32 accumulation), then  P(fp64) -= D  in the epilogue.  There is no fp64 kind of wgmma, so this
// path is the "fp32 covariance" mode of SURVEY.md §8d (config 3): the correction carries fp32 accuracy,
// P itself stays fp64 in HBM so every other kernel is unchanged.  It is opt-in ("covariance_update":
// "tf32x3" in the estimator config, or flags bit 0 of xivo_ekf_update_ex); the default remains fp64.
//
// One CTA (128 threads = one warpgroup; two m64 MMAs cover the 128 rows) per (filter, 128-row tile, 32-column
// chunk) of the upper triangle (narrow chunks: the tile is latency-, not math-bound, so more CTAs per filter win).
// Operands are staged by the CTA's threads (fp64 -> hi/lo TF32, transposed) into the canonical K-major no-swizzle
// shared-memory layout of the wgmma matrix descriptor: 8-row x 16-byte core matrices,
//   byte(row, k) = ((k / 4) * ROWS + row) * 16 + (k % 4) * 4
// i.e. SBO (8-row group stride) = 128 B and LBO (stride between the two 16-byte K chunks of one MMA) =
// ROWS * 16 B.  K (= measurement rows) is consumed in blocks of 32 (four K=8 MMAs per pass).
#include <atomic>
#include <cstdint>
#include <cstdlib>

#include "kernels.h"
#include "prof.h"

namespace xb {
namespace {

constexpr int TC_MT = 128;       // rows per tile = two m64 MMAs of one warpgroup
constexpr int TC_NT = 32;        // columns per chunk: narrow chunks = more CTAs per filter (the tile work is latency, not math)
constexpr int TC_KB = 32;        // K elements staged per block
constexpr int TC_THREADS = 128;

__device__ int g_tc_fault;  // set when an mbarrier wait timed out (never expected; keeps a bad build from hanging the GPU)

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ uint32_t to_tf32(float x) {
  uint32_t r;
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(r) : "f"(x));
  return r;
}

// wgmma shared-memory matrix descriptor (sm_90): start address, LBO, SBO in 16-byte units, base offset 0,
// layout type 0 (no swizzle).
__device__ __forceinline__ uint64_t gmma_smem_desc(uint32_t saddr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
  uint64_t d = 0;
  d |= (uint64_t)((saddr & 0x3FFFFu) >> 4);
  d |= (uint64_t)((lbo_bytes >> 4) & 0x3FFFu) << 16;
  d |= (uint64_t)((sbo_bytes >> 4) & 0x3FFFu) << 32;
  return d;
}

// D(64 x 32, fp32, registers) (+)= A(64 x 8, TF32, K-major) * B(32 x 8, TF32, K-major)^T.  Accumulator fragment:
// d[4 i + 2 h + e] = D[16 (warp % 4) + lane / 4 + 8 h][8 i + 2 (lane % 4) + e].
__device__ __forceinline__ void wgmma_tf32_m64n32(float (&d)[16], uint64_t da, uint64_t db, uint32_t accumulate) {
  asm volatile(
      "{\n\t"
      ".reg .pred p;\n\t"
      "setp.ne.b32 p, %18, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n32k8.f32.tf32.tf32 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, %16, %17, p, 1, 1;\n\t"
      "}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]),
        "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
      : "l"(da), "l"(db), "r"(accumulate));
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_wait_all() { asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory"); }
// keeps the compiler from moving accesses of the accumulator registers across the asynchronous MMAs
__device__ __forceinline__ void acc_fence(float (&d)[16]) {
#pragma unroll
  for (int i = 0; i < 16; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// four consecutive k of one row -> 16-byte chunk `chunk` of the hi array and of the lo array (x = hi + lo, both TF32)
__device__ __forceinline__ void stage_chunk(const double (&x)[4], uint32_t* hi, uint32_t* lo, int chunk) {
  uint4 h, l;
  uint32_t* hp = &h.x;
  uint32_t* lp = &l.x;
#pragma unroll
  for (int q = 0; q < 4; ++q) {
    const uint32_t t = to_tf32((float)x[q]);
    hp[q] = t;
    lp[q] = to_tf32((float)(x[q] - (double)__uint_as_float(t)));
  }
  reinterpret_cast<uint4*>(hi)[chunk] = h;
  reinterpret_cast<uint4*>(lo)[chunk] = l;
}

__global__ void __launch_bounds__(TC_THREADS) ekf_cov_tc_kernel(int N, const int* __restrict__ nsel, int Mdense, int Mmax,
                                                                const double* __restrict__ HP, const double* __restrict__ Kt,
                                                                double* __restrict__ P) {
  extern __shared__ __align__(128) unsigned char tc_smem[];

  const int b = blockIdx.z;
  const int M = nsel ? 2 * nsel[b] : Mdense;
  const int m0 = blockIdx.y * TC_MT;
  const int n0 = m0 + blockIdx.x * TC_NT;  // only the upper triangle: columns start at the tile's first row
  if (M == 0 || m0 >= N || n0 >= N) return;  // uniform over the CTA
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;

  uint32_t* Ah = reinterpret_cast<uint32_t*>(tc_smem);
  uint32_t* Al = Ah + TC_KB * TC_MT;
  uint32_t* Bh = Al + TC_KB * TC_MT;
  uint32_t* Bl = Bh + TC_KB * TC_NT;
  const double* __restrict__ HPb = HP + (size_t)b * Mmax * N;
  const double* __restrict__ Ktb = Kt + (size_t)b * Mmax * N;
  double* __restrict__ Pb = P + (size_t)b * N * N;

  const uint32_t a_chunk = TC_MT * 16, b_chunk = TC_NT * 16;  // bytes between consecutive 16-byte K chunks
  const int nkb = (M + TC_KB - 1) / TC_KB;
  float acc[2][16];  // rows 0-63 and 64-127 of the tile
#pragma unroll
  for (int i = 0; i < 16; ++i) acc[0][i] = acc[1][i] = 0.f;

  for (int kb = 0; kb < nkb; ++kb) {
    const int k0 = kb * TC_KB;
    // ---- stage A(i, k) = Kt[k][m0 + i] and B(j, k) = HP[k][n0 + j] as hi/lo TF32, zero padded.  A thread owns one row and
    // converts four consecutive k at a time: four coalesced loads -> one 16-byte chunk of the hi array and one of the lo array.
    const int kreal = min(TC_KB, M - k0);
    const int kgroups = ((kreal + 7) >> 3) << 1;  // 16-byte chunks the MMAs of this block read
    {
      const int gi = m0 + tid;
      const double* __restrict__ src = Ktb + (size_t)k0 * N + gi;
#pragma unroll 2
      for (int g = 0; g < kgroups; ++g) {
        double x[4];
#pragma unroll
        for (int q = 0; q < 4; ++q) x[q] = (gi < N && 4 * g + q < kreal) ? src[(size_t)(4 * g + q) * N] : 0.0;
        stage_chunk(x, Ah, Al, g * TC_MT + tid);
      }
    }
    for (int u = tid; u < kgroups * TC_NT; u += TC_THREADS) {  // 32 rows: the k groups are spread over the warps
      const int g = u / TC_NT, r = u - g * TC_NT;
      const int gj = n0 + r;
      const double* __restrict__ src = HPb + (size_t)k0 * N + gj;
      double x[4];
#pragma unroll
      for (int q = 0; q < 4; ++q) x[q] = (gj < N && 4 * g + q < kreal) ? src[(size_t)(4 * g + q) * N] : 0.0;
      stage_chunk(x, Bh, Bl, g * TC_NT + r);
    }
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");  // generic-proxy writes -> visible to the tensor core (async proxy)
    __syncthreads();
    const int ksteps = kgroups >> 1;  // K = 8 per tf32 MMA; all-zero steps are skipped
    const uint32_t aH = smem_u32(Ah), aL = smem_u32(Al), bH = smem_u32(Bh), bL = smem_u32(Bl);
    acc_fence(acc[0]);
    acc_fence(acc[1]);
    wgmma_fence();
#pragma unroll 1
    for (int pass = 0; pass < 3; ++pass) {  // small terms first
      const uint32_t sa = pass == 0 ? aL : aH, sb = pass == 1 ? bL : bH;
#pragma unroll 1
      for (int ks = 0; ks < ksteps; ++ks) {
        const uint64_t db = gmma_smem_desc(sb + (uint32_t)ks * 2u * b_chunk, b_chunk, 128u);
        wgmma_tf32_m64n32(acc[0], gmma_smem_desc(sa + (uint32_t)ks * 2u * a_chunk, a_chunk, 128u), db, 1u);
        wgmma_tf32_m64n32(acc[1], gmma_smem_desc(sa + (uint32_t)ks * 2u * a_chunk + 64u * 16u, a_chunk, 128u), db, 1u);
      }
    }
    wgmma_commit();
    wgmma_wait_all();
    acc_fence(acc[0]);
    acc_fence(acc[1]);
    __syncthreads();  // every warp's MMAs are complete before the operands are overwritten
  }

  // ---- epilogue: P -= D on the upper triangle, mirrored
#pragma unroll
  for (int h = 0; h < 2; ++h)
#pragma unroll
    for (int v = 0; v < 16; ++v) {
      const int row = m0 + h * 64 + warp * 16 + (lane >> 2) + 8 * ((v >> 1) & 1);
      const int col = n0 + 8 * (v >> 2) + 2 * (lane & 3) + (v & 1);
      if (row < N && col < N && col >= row) {
        const double val = Pb[(size_t)row * N + col] - (double)acc[h][v];
        Pb[(size_t)row * N + col] = val;
        if (col != row) Pb[(size_t)col * N + row] = val;
      }
    }
}


// ------------------------------------------------------------------------------------------------------------------------------
// Second formulation (default for "covariance_update": "tf32x3"; XIVO_TC_V1=1 keeps the kernel above for A/B parity).
// What changed and why (the first kernel spends its time staging operands, not in the tensor cores):
//  * operands are not converted here: the gain kernel, which owns one state column per thread when it finishes K^T, writes K^T and HP
//    once more as TF32 hi/lo words directly in the canonical K-major layout  [filter][hi|lo][k/4][state column][4 words]
//    (column stride 16 B = one core-matrix row, 8 columns = one 128-byte core matrix, k-chunk stride = Npad * 16 B);
//  * a CTA owns a 128-row tile of one filter and walks ALL its 32-column chunks of the upper triangle: the A operand (128 rows x
//    all K, hi and lo) arrives once by TMA box loads {4, 128, 8} and stays in shared memory, the B chunks {4, 32, 8} are double
//    buffered and prefetched two chunks ahead;
//  * warpgroups 0 and 1 each own 64 rows of the tile and keep their fp32 accumulator in registers; the MMAs of chunk i+1 are issued
//    asynchronously before the epilogue of chunk i streams P;
//  * the epilogue goes through shared memory so that both the direct update P[i][j] and the mirrored one P[j][i] are row-contiguous
//    (the first kernel writes 8-byte words 8 N bytes apart).  The mirrored element is recomputed from its own old value, which equals
//    P[i][j] bit for bit because P is kept exactly symmetric, so it stays exactly symmetric.
// The contraction is bound by the fp64 traffic of P (2 N^2 8 B per filter against 3 * 2 N^2 M flop): see DESIGN.md section 4.
constexpr int T2_MT = 128, T2_NT = 32, T2_KB = 32, T2_THREADS = 512;  // warpgroups 0-1 run the MMAs; all 16 warps stream P in the epilogue
constexpr int T2_A_BLOCK = (T2_KB / 4) * T2_MT * 16;  // bytes of one k-block of A (hi or lo): 8 chunks x 128 rows x 16 B = 16 KB
constexpr int T2_B_BLOCK = (T2_KB / 4) * T2_NT * 16;  // 4 KB

__device__ __forceinline__ bool mbar_wait(uint32_t addr, uint32_t parity) {  // bounded (a broken build must not hang the device)
  uint32_t done = 0;
  const long long t0 = clock64();
  while (!done) {
    asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}" : "=r"(done) : "r"(addr), "r"(parity) : "memory");
    if (!done && clock64() - t0 > 400000000LL) return false;
  }
  return true;
}
__device__ __forceinline__ void tma_box3(uint32_t dst, const CUtensorMap* map, int c0, int c1, int c2, uint32_t bar) {
  asm volatile("cp.async.bulk.tensor.3d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3, %4}], [%5];"
               ::"r"(dst), "l"(reinterpret_cast<unsigned long long>(map)), "r"(c0), "r"(c1), "r"(c2), "r"(bar) : "memory");
}

__global__ void __launch_bounds__(T2_THREADS) ekf_cov_tc2_kernel(const __grid_constant__ CUtensorMap mapA, const __grid_constant__ CUtensorMap mapB, int N,
                                                                 const int* __restrict__ nsel, int Mdense, int KCmax, double* __restrict__ P) {
  extern __shared__ __align__(128) unsigned char t2_smem[];
  __shared__ __align__(8) unsigned long long bars[3];  // 0: A landed; 1, 2: B buffer landed
  const int b = blockIdx.y, m0 = blockIdx.x * T2_MT;
  const int M = nsel ? 2 * nsel[b] : Mdense;
  if (M == 0 || m0 >= N) return;  // uniform over the CTA
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int wg = __shfl_sync(0xffffffffu, warp >> 2, 0);  // warp-uniform in the compiler's view: the MMAs below are not serialized
  const int kblocks = (M + T2_KB - 1) / T2_KB;
  const int kbmax = KCmax / (T2_KB / 4);
  // shared: A hi [kbmax][16 KB] | A lo | B buffers 2 x (hi [kbmax][4 KB] | lo) | D staging 128 x 33 floats
  unsigned char* sAh = t2_smem;
  unsigned char* sAl = sAh + (size_t)kbmax * T2_A_BLOCK;
  unsigned char* sB = sAl + (size_t)kbmax * T2_A_BLOCK;
  const uint32_t b_buf_bytes = (uint32_t)kbmax * 2u * T2_B_BLOCK;
  float* sD = reinterpret_cast<float*>(sB + 2 * (size_t)b_buf_bytes);
  const uint32_t barA = smem_u32(&bars[0]);
  if (tid == 0) {
    for (int i = 0; i < 3; ++i) asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(smem_u32(&bars[i])) : "memory");
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  const int ncc = (N - m0 + T2_NT - 1) / T2_NT;                // column chunks of this row tile: columns [m0, N)
  const int zA = (b * 2) * KCmax, zB = zA;                      // first k-chunk of filter b's hi slab inside the maps (lo slab: + KCmax)
  auto load_b = [&](int chunk) {                                // thread 0: TMA of column chunk `chunk` into buffer chunk & 1
    const int buf = chunk & 1;
    const uint32_t bar = smem_u32(&bars[1 + buf]);
    const uint32_t dst = smem_u32(sB) + (uint32_t)buf * b_buf_bytes;
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"((uint32_t)kblocks * 2u * T2_B_BLOCK) : "memory");
    for (int kb = 0; kb < kblocks; ++kb) {
      tma_box3(dst + (uint32_t)kb * T2_B_BLOCK, &mapB, 0, m0 + chunk * T2_NT, zB + kb * (T2_KB / 4), bar);
      tma_box3(dst + (uint32_t)(kbmax + kb) * T2_B_BLOCK, &mapB, 0, m0 + chunk * T2_NT, zB + KCmax + kb * (T2_KB / 4), bar);
    }
  };
  float acc[16];  // written first by an MMA with the accumulator input disabled
  auto issue_mma = [&](int chunk) {                             // warpgroups 0, 1: 3 passes x kblocks x 4 MMAs into acc, one commit group
    const int buf = chunk & 1;
    const uint32_t bH = smem_u32(sB) + (uint32_t)buf * b_buf_bytes, bL = bH + (uint32_t)kbmax * T2_B_BLOCK;
    const uint32_t aH = smem_u32(sAh) + (uint32_t)wg * 64u * 16u, aL = smem_u32(sAl) + (uint32_t)wg * 64u * 16u;
    uint32_t first = 1;
    acc_fence(acc);
    wgmma_fence();
#pragma unroll 1
    for (int pass = 0; pass < 3; ++pass) {                      // small terms first: lo*hi, hi*lo, hi*hi
      const uint32_t sa = pass == 0 ? aL : aH, sb = pass == 1 ? bL : bH;
#pragma unroll 1
      for (int kb = 0; kb < kblocks; ++kb) {
        const int ksteps = min(T2_KB / 8, (M - kb * T2_KB + 7) / 8);  // K = 8 per MMA; all-zero tail steps are skipped
#pragma unroll 1
        for (int ks = 0; ks < ksteps; ++ks) {
          const uint64_t da = gmma_smem_desc(sa + (uint32_t)kb * T2_A_BLOCK + (uint32_t)ks * 2u * (T2_MT * 16), T2_MT * 16, 128u);
          const uint64_t db = gmma_smem_desc(sb + (uint32_t)kb * T2_B_BLOCK + (uint32_t)ks * 2u * (T2_NT * 16), T2_NT * 16, 128u);
          wgmma_tf32_m64n32(acc, da, db, first ? 0u : 1u);
          first = 0;
        }
      }
    }
    wgmma_commit();
  };
  if (tid == 0) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(barA), "r"((uint32_t)kblocks * 2u * T2_A_BLOCK) : "memory");
    for (int kb = 0; kb < kblocks; ++kb) {
      tma_box3(smem_u32(sAh) + (uint32_t)kb * T2_A_BLOCK, &mapA, 0, m0, zA + kb * (T2_KB / 4), barA);
      tma_box3(smem_u32(sAl) + (uint32_t)kb * T2_A_BLOCK, &mapA, 0, m0, zA + KCmax + kb * (T2_KB / 4), barA);
    }
    load_b(0);
    if (ncc > 1) load_b(1);
  }
  // every thread sees the operands land and the CTA agrees on the outcome, so the warpgroup-wide MMAs are never divergent
  bool fault = !__syncthreads_and(mbar_wait(barA, 0u) && mbar_wait(smem_u32(&bars[1]), 0u));
  if (!fault && wg < 2) issue_mma(0);
  double* __restrict__ Pb = P + (size_t)b * N * N;
  for (int i = 0; i < ncc && !fault; ++i) {
    if (wg < 2) {
      // chunk i complete -> shared staging (row stride 33 floats)
      wgmma_wait_all();
      acc_fence(acc);
      const int r0 = wg * 64 + (warp & 3) * 16 + (lane >> 2), c0 = 2 * (lane & 3);
#pragma unroll
      for (int v = 0; v < 16; ++v) sD[(r0 + 8 * ((v >> 1) & 1)) * (T2_NT + 1) + c0 + 8 * (v >> 2) + (v & 1)] = acc[v];
    }
    // staging complete, B buffer i & 1 no longer read, B chunk i + 1 landed
    const bool landed = i + 1 >= ncc || mbar_wait(smem_u32(&bars[1 + ((i + 1) & 1)]), (uint32_t)((i + 1) >> 1) & 1u);
    if (!__syncthreads_and(landed)) {
      fault = true;
      break;
    }
    if (wg < 2 && i + 1 < ncc) issue_mma(i + 1);                 // next chunk's MMAs run while this chunk's epilogue does
    if (tid == 0 && i + 2 < ncc) load_b(i + 2);
    const int n0 = m0 + i * T2_NT;
    // 4096 tile elements, 512 threads: every thread issues its 8 + 8 loads of P before the first dependent store, so that the SM keeps
    // ~8 K loads in flight (one load per thread at a time runs at a few percent of the HBM rate).
    constexpr int PER = T2_MT * T2_NT / T2_THREADS;
    double pv[PER];
    size_t po[PER];
    float dv[PER];
    // direct part: P[m0 + r][n0 + c] for r <= c (global indices), 32 consecutive doubles per row
#pragma unroll
    for (int k = 0; k < PER; ++k) {
      const int idx = tid + k * T2_THREADS;
      const int r = idx >> 5, c = idx & 31;
      const int gi = m0 + r, gj = n0 + c;
      const bool on = gi < N && gj < N && gi <= gj;
      po[k] = on ? (size_t)gi * N + gj : ~(size_t)0;
      dv[k] = sD[r * (T2_NT + 1) + c];
      pv[k] = on ? Pb[po[k]] : 0.0;
    }
#pragma unroll
    for (int k = 0; k < PER; ++k)
      if (po[k] != ~(size_t)0) Pb[po[k]] = pv[k] - (double)dv[k];
    // mirrored part: P[n0 + c][m0 + r] for r < c, 128 consecutive doubles per row; the old value read here equals P[m0 + r][n0 + c]
#pragma unroll
    for (int k = 0; k < PER; ++k) {
      const int idx = tid + k * T2_THREADS;
      const int c = idx >> 7, r = idx & 127;
      const int gi = m0 + r, gj = n0 + c;
      const bool on = gi < N && gj < N && gi < gj;
      po[k] = on ? (size_t)gj * N + gi : ~(size_t)0;
      dv[k] = sD[r * (T2_NT + 1) + c];
      pv[k] = on ? Pb[po[k]] : 0.0;
    }
#pragma unroll
    for (int k = 0; k < PER; ++k)
      if (po[k] != ~(size_t)0) Pb[po[k]] = pv[k] - (double)dv[k];
    __syncthreads();                                            // staging is free again
  }
  if (fault && tid == 0) atomicExch(&g_tc_fault, 1);
}

}  // namespace

size_t ekf_cov_tc_smem() { return (size_t)2 * TC_KB * (TC_MT + TC_NT) * sizeof(uint32_t); }

int launch_ekf_cov_tc(cudaStream_t st, int N, const int* nsel, int Mdense, int Mmax, const double* HP, const double* Kt, double* P,
                      int batch) {
  const size_t smem = ekf_cov_tc_smem();
  XB_CUDA(cudaFuncSetAttribute(ekf_cov_tc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  const int tm = (N + TC_MT - 1) / TC_MT, tn = (N + TC_NT - 1) / TC_NT;
  ProfScope ps("ekf_cov", st);
  ekf_cov_tc_kernel<<<dim3(tn, tm, batch), TC_THREADS, smem, st>>>(N, nsel, Mdense, Mmax, HP, Kt, P);
  XB_CUDA(cudaGetLastError());
  return 0;
}

// ---- operand buffers of the second formulation -------------------------------------------------------------------------------
int tc_npad(int N) { return (N + 7) & ~7; }
int tc_kcmax(int Mmax) { return ((Mmax + T2_KB - 1) / T2_KB) * (T2_KB / 4); }
size_t tc_operand_words(int N, int Mmax, int batch) { return (size_t)batch * 2 * tc_kcmax(Mmax) * tc_npad(N) * 4; }

static int make_operand_map(CUtensorMap* out, const uint32_t* base, int Npad, int KCmax, int batch, int box_rows) {
  typedef CUresult (*EncodeFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*, const cuuint32_t*,
                               const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
  static EncodeFn encode = nullptr;
  if (!encode) {
    void* fn = nullptr;
    cudaDriverEntryPointQueryResult q;
    XB_CUDA(cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &q));
    XB_REQUIRE(fn && q == cudaDriverEntryPointSuccess, "cuTensorMapEncodeTiled is not available from this driver");
    encode = reinterpret_cast<EncodeFn>(fn);
  }
  // {4 words, state column, k-chunk of (filter, hi|lo)}: column stride 16 B, chunk stride Npad * 16 B
  const cuuint64_t dims[3] = {4, (cuuint64_t)Npad, (cuuint64_t)batch * 2 * KCmax};
  const cuuint64_t strides[2] = {16, (cuuint64_t)Npad * 16};
  const cuuint32_t box[3] = {4, (cuuint32_t)box_rows, (cuuint32_t)(T2_KB / 4)};
  const cuuint32_t estr[3] = {1, 1, 1};
  const CUresult r = encode(out, CU_TENSOR_MAP_DATA_TYPE_UINT32, 3, const_cast<uint32_t*>(base), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                            CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  XB_REQUIRE(r == CUDA_SUCCESS, "cuTensorMapEncodeTiled failed for the update operands");
  return 0;
}

int tc_operands_init(TcOperands* t, int N, int Mmax, int batch, uint32_t* kt32, uint32_t* hp32) {
  t->kt32 = kt32; t->hp32 = hp32;
  t->Npad = tc_npad(N); t->KCmax = tc_kcmax(Mmax); t->batch = batch;
  if (int rc = make_operand_map(&t->mapA, kt32, t->Npad, t->KCmax, batch, T2_MT)) return rc;
  return make_operand_map(&t->mapB, hp32, t->Npad, t->KCmax, batch, T2_NT);
}

size_t ekf_cov_tc2_smem(int KCmax) {
  const size_t kbmax = (size_t)KCmax / (T2_KB / 4);
  return kbmax * 2 * T2_A_BLOCK + 2 * kbmax * 2 * T2_B_BLOCK + (size_t)T2_MT * (T2_NT + 1) * sizeof(float);
}

int ekf_cov_tc2_max_rows() {
  int m = 0;
  while (ekf_cov_tc2_smem(tc_kcmax(m + 1)) <= kSmemOptin) ++m;
  return m;
}

int launch_ekf_cov_tc2(cudaStream_t st, int N, const int* nsel, int Mdense, const TcOperands& t, double* P, int batch) {
  XB_REQUIRE(t.KCmax <= tc_kcmax(ekf_cov_tc2_max_rows()), "tensor-core downdate: measurement dimension too large for the resident A operand");
  const size_t smem = ekf_cov_tc2_smem(t.KCmax);
  XB_REQUIRE(batch <= t.batch, "tensor-core downdate: operand buffers hold fewer filters");
  static std::atomic<size_t> attr{0};
  if (smem > attr.load(std::memory_order_relaxed)) {
    XB_CUDA(cudaFuncSetAttribute(ekf_cov_tc2_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    attr.store(smem, std::memory_order_relaxed);
  }
  ProfScope ps("ekf_cov", st);
  ekf_cov_tc2_kernel<<<dim3((N + T2_MT - 1) / T2_MT, batch), T2_THREADS, smem, st>>>(t.mapA, t.mapB, N, nsel, Mdense, t.KCmax, P);
  XB_CUDA(cudaGetLastError());
  return 0;
}

int ekf_cov_tc_fault(cudaStream_t st) {
  int f = 0;
  if (cudaMemcpyFromSymbolAsync(&f, g_tc_fault, sizeof(int), 0, cudaMemcpyDeviceToHost, st) != cudaSuccess) return -1;
  if (cudaStreamSynchronize(st) != cudaSuccess) return -1;
  return f;
}

}  // namespace xb
