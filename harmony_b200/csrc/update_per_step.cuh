// update_per_step.cuh — harmony::update_R (harmony.cpp:269-342) as three launches per block step: column sums of
// the block's current R, the table update, and the block's new R.  It serves every shape the persistent kernels
// cannot take (K > 256, rings or tables that do not fit shared memory), calls of more rounds than the two-pass
// kernel's R-store mask holds, and the legacy centroid step.
#pragma once
#include "kernels.cuh"

namespace hb {

// ------------------------------------------------------------------------------------------------
// update_R block step (harmony.cpp:293-332)
// ------------------------------------------------------------------------------------------------
struct StepArgs {
  const float* U;
  float* R;
  const int* order;         // [n] cells sorted by (block, tuple, cell)
  const int* seg_start;     // [nb*J + 1]
  const int* tile_base;     // [nb*J + 1] exclusive scan of tiles per segment
  const int* tuple_levels;  // [J][C]
  const float* sigma;
  const float* P;           // [B][K] penalty table of this step
  float* acc_O;             // [B][K] column sums per level (rem_j or add_j)
  float* acc_rs;            // [K]
  double* obj_acc;          // [2]
  int blk, J, K, C, KP, KS;
};

// tile -> (segment, first position, length)
__device__ __forceinline__ bool locate_tile(const StepArgs& a, int t, int* sh_info) {
  // sh_info: [0] seg, [1] p0, [2] len, [3] valid
  if (threadIdx.x == 0) {
    int s_lo = a.blk * a.J, s_hi = (a.blk + 1) * a.J;
    int t0 = a.tile_base[s_lo], t1 = a.tile_base[s_hi];
    int tt = t0 + t;
    if (tt >= t1) {
      sh_info[3] = 0;
    } else {
      int lo = s_lo, hi = s_hi;  // find the last seg with tile_base[seg] <= tt
      while (hi - lo > 1) {
        int mid = (lo + hi) >> 1;
        if (a.tile_base[mid] <= tt) lo = mid; else hi = mid;
      }
      int p0 = a.seg_start[lo] + (tt - a.tile_base[lo]) * TM;
      int len = a.seg_start[lo + 1] - p0;
      sh_info[0] = lo;
      sh_info[1] = p0;
      sh_info[2] = len < TM ? len : TM;
      sh_info[3] = 1;
    }
  }
  __syncthreads();
  return sh_info[3] != 0;
}

// Step 1 (:312-313): column sums of the block's current R, per level  ->  acc_O / acc_rs
template <int KQ>
__global__ void __launch_bounds__(ROW_THREADS) k_block_colsum(StepArgs a) {
  extern __shared__ __align__(16) float smem[];
  __shared__ int info[4];
  const int K = a.K, KP = a.KP;
  float* part = smem;  // [NWARP][KP]
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  for (int t = blockIdx.x;; t += gridDim.x) {
    __syncthreads();
    if (!locate_tile(a, t, info)) break;
    const int seg = info[0], p0 = info[1], len = info[2];
    const int q = seg - a.blk * a.J;
    float cs[KQ];
#pragma unroll
    for (int qq = 0; qq < KQ; ++qq) cs[qq] = 0.f;
    for (int r = warp; r < len; r += NWARP) {
      const size_t row = (size_t)a.order[p0 + r];
#pragma unroll
      for (int qq = 0; qq < KQ; ++qq) {
        int k = lane + 32 * qq;
        if (k < K) cs[qq] += a.R[row * a.KS + k];
      }
    }
#pragma unroll
    for (int qq = 0; qq < KQ; ++qq) {
      int k = lane + 32 * qq;
      if (k < KP) part[warp * KP + k] = cs[qq];
    }
    __syncthreads();
    for (int k = tid; k < K; k += ROW_THREADS) {
      float s = 0.f;
#pragma unroll
      for (int w = 0; w < NWARP; ++w) s += part[w * KP + k];
      atomicAdd(a.acc_rs + k, s);
      for (int c = 0; c < a.C; ++c) atomicAdd(a.acc_O + (size_t)a.tuple_levels[q * a.C + c] * a.KS + k, s);
    }
  }
}

// Finish step j-1 and start step j on the K x B tables:
//   O += add_prev; E += rs_add_prev*Pr_b        (:329-330 of the previous block)
//   O -= rem;      E -= rs_rem*Pr_b             (:312-313 of this block)
//   P = ((2E+1)/(O+E+1))^theta                  (:322, harmony_pow utils.cpp:84-90)
// add_prev / rem may be null (first step of a round / finalisation after the last step).
__global__ void k_step_prepare(float* __restrict__ O, float* __restrict__ E, const float* __restrict__ add_O,
                               const float* __restrict__ add_rs, const float* __restrict__ rem_O,
                               const float* __restrict__ rem_rs, const float* __restrict__ Pr_b,
                               const float* __restrict__ theta, float* __restrict__ P, int B, int K, int KS) {
  int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= B * KS) return;
  int b = idx / KS, k = idx - b * KS;
  if (k >= K) return;
  float o = O[idx], e = E[idx];
  if (add_O) {
    e += add_rs[k] * Pr_b[b];
    o += add_O[idx];
  }
  if (rem_O) {
    e -= rem_rs[k] * Pr_b[b];
    o -= rem_O[idx];
  }
  O[idx] = o;
  E[idx] = e;
  if (P) P[idx] = powf(((2.f * e) + 1.f) / (o + e + 1.f), theta[b]);
}

// Step 2+3 (:318-330): R = L1norm(exp(U) * sum_c P[level_c]), column sums of the new R -> acc_O/acc_rs,
// objective partials of the new R.
template <int KQ>
__global__ void __launch_bounds__(ROW_THREADS) k_block_update(StepArgs a) {
  extern __shared__ __align__(16) float smem[];
  __shared__ int info[4];
  const int K = a.K, KP = a.KP;
  float* part = smem;             // [NWARP][KP]
  float* Psum = part + NWARP * KP;  // [KP]
  float* lP = Psum + KP;          // [KP]
  float* sig = lP + KP;           // [KP]
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  for (int k = tid; k < KP; k += ROW_THREADS) sig[k] = (k < K) ? a.sigma[k] : 1.f;
  float okd = 0.f, oent = 0.f;
  for (int t = blockIdx.x;; t += gridDim.x) {
    __syncthreads();
    if (!locate_tile(a, t, info)) break;
    const int seg = info[0], p0 = info[1], len = info[2];
    const int q = seg - a.blk * a.J;
    for (int k = tid; k < K; k += ROW_THREADS) {
      float s = 0.f;
      for (int c = 0; c < a.C; ++c) s += a.P[(size_t)a.tuple_levels[q * a.C + c] * a.KS + k];
      Psum[k] = s;
      lP[k] = logf(s);
    }
    __syncthreads();
    float cs[KQ];
#pragma unroll
    for (int qq = 0; qq < KQ; ++qq) cs[qq] = 0.f;
    for (int r = warp; r < len; r += NWARP) {
      const size_t row = (size_t)a.order[p0 + r];
      float u[KQ], e[KQ];
      float s = 0.f;
#pragma unroll
      for (int qq = 0; qq < KQ; ++qq) {
        int k = lane + 32 * qq;
        if (k < K) {
          u[qq] = ld_stream(a.U + row * a.KS + k);
          e[qq] = expf(u[qq]) * Psum[k];
        } else {
          u[qq] = 0.f;
          e[qq] = 0.f;
        }
        s += fabsf(e[qq]);
      }
      s = warp_sum(s);
      const float sdiv = (s == 0.f) ? 1.f : s;  // arma::normalise(.., 1, 0): zero norm divides by 1
      const float ls = logf(sdiv);
#pragma unroll
      for (int qq = 0; qq < KQ; ++qq) {
        int k = lane + 32 * qq;
        if (k < K) {
          float rv = e[qq] / sdiv;
          st_stream(a.R + row * a.KS + k, rv);
          cs[qq] += rv;
          okd += rv * (-sig[k] * u[qq]);
          if (rv > 0.f) oent += sig[k] * rv * (u[qq] + lP[k] - ls);
        }
      }
    }
#pragma unroll
    for (int qq = 0; qq < KQ; ++qq) {
      int k = lane + 32 * qq;
      if (k < KP) part[warp * KP + k] = cs[qq];
    }
    __syncthreads();
    for (int k = tid; k < K; k += ROW_THREADS) {
      float s = 0.f;
#pragma unroll
      for (int w = 0; w < NWARP; ++w) s += part[w * KP + k];
      atomicAdd(a.acc_rs + k, s);
      for (int c = 0; c < a.C; ++c) atomicAdd(a.acc_O + (size_t)a.tuple_levels[q * a.C + c] * a.KS + k, s);
    }
  }
  okd = warp_sum(okd);
  oent = warp_sum(oent);
  if (lane == 0) {
    atomicAdd(a.obj_acc + 0, (double)okd);
    atomicAdd(a.obj_acc + 1, (double)oent);
  }
}

}  // namespace hb
