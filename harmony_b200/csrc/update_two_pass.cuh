// update_two_pass.cuh — persistent cooperative kernel for harmony::update_R (harmony.cpp:269-342) that reads every
// U row twice per round (the second read hits L2).  Up to K = 256 it serves the shapes the single-pass kernel
// (update_single_pass.cuh) cannot take: 2 J > #SMs (a CTA's slice of a block spans several tuples), or n KS >= 2^32.
//
// One launch covers a range of global block steps s = round * nb + block of one cluster_cpp call.  Steps
// are separated by a grid-wide barrier (the Gauss-Seidel dependency on O, E).  Each CTA has two warp
// groups that run concurrently within step s:
//   group U  updates its share of the rows of block s:   R = L1norm(exp(U) * sum_c P_s[level_c])   (:318-323)
//            accumulating the new column sums per level (add_s, :329-330) and the objective partials;
//            its first CTAs also materialise the K x B tables O_s, E_s and save the penalty table P_s;
//   group L  looks ahead: the column sums of the *current* R of its share of block s+1 (rem_{s+1},
//            :312-313), recomputed from U and the penalty tables of the previous round (R itself is only
//            stored in the rounds after which cluster_cpp may return).
// HBM traffic per cell and round: one read of the U row (its second touch, one step later, hits L2).
// Row loads are software-pipelined (the next batch is in flight while the current one is reduced) and
// are issued before the step's tables are derived, so the table latency hides behind them.
//
// Per-step accumulator slots and the derivation of the step tables: update_slots.cuh.
#pragma once
#include <type_traits>

#include "update_slots.cuh"

namespace hb {

constexpr int UPD_THREADS = 1024;
constexpr int UPD_GROUP = 512;               // threads per warp group
constexpr int UPD_GWARPS = UPD_GROUP / 32;   // warps per group
constexpr int UPD_LPR = 16;                  // lanes per row
constexpr int UPD_RPW = 32 / UPD_LPR;        // rows per warp
constexpr int UPD_BATCH = UPD_GWARPS * UPD_RPW;  // rows per batch per group
constexpr int UPD_STAGE = 2048;              // staged order entries per group
// cp.async stages per warp: the look-ahead group streams from HBM (deep), the update group re-reads from L2
__host__ __device__ constexpr int upd_depth_look(int nv) { return nv <= 2 ? 8 : 2; }
__host__ __device__ constexpr int upd_depth_upd(int nv) { return nv <= 2 ? 4 : 2; }
constexpr int UPD_RUNAHEAD = 3;              // block steps the look-ahead group may run ahead of the update group

struct TwoPassArgs {
  const float* U;   // [n][KS]
  float* R;         // [n][KS]
  const int* order;      // [T][n]   rows sorted by (block, tuple, cell) per round
  const int* prev_at;    // [T][n]   block (in the previous round) of the cell at each position of `order`
  const int* seg_start;  // [T][nb*J + 1]
  const int4* ranges;    // [T*nb][grid] (lo, hi, tuple, 0): tuple-aligned CTA ranges, or null (even split)
  const int* tuple_levels;  // [J][C]
  const float* sigma;    // [K]
  const float* theta;    // [B]
  const float* Pr_b;     // [B]
  float* ring;           // [2 parity][2 (O,E)][B][KS]
  float* acc;            // [(S+2)][SL]  slot(s) at (s+1)*SL: [addprev_O B*KS | addprev_rs KS | rem_O B*KS | rem_rs KS]
  float* Psave;          // [2 round parity][nb][B][KS]
  float* OEend;          // [T][2][B][KS]  tables at the end of each round (for the objective)
  double* obj;           // [T][2]
  unsigned* bar;         // [2][S + 2] completion counters: cntU[s + 1], cntL[s + 1] = #CTAs done with step s
  int64_t n;
  int K, KS, C, J, B, nb, T;
  int s_begin, s_end;    // steps [s_begin, s_end)
  int prologue;          // run the look-ahead for s_begin before the first step (then barrier)
  int first_round_from_R;  // look-ahead of round 0 reads R from memory (R was written by the user)
  unsigned write_R_mask;   // bit t: store R in round t
  int sigma_uniform;       // all sigma_k equal sigma0 (the default: scalar sigma)
  float sigma0;
  int use_barrier;         // 0 when the launch covers a single step and no prologue (no co-residency needed)
};

__device__ __forceinline__ void group_sync(int id) { asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(UPD_GROUP) : "memory"); }

enum { MODE_UPDATE = 0, MODE_LOOK_U = 1, MODE_LOOK_R = 2 };

// NV = float4 per lane (UPD_LPR lanes per row): K <= 4 * UPD_LPR * NV
template <int NV>
__global__ void __launch_bounds__(UPD_THREADS, 1) k_update_two_pass(TwoPassArgs a) {
  extern __shared__ __align__(16) float smem[];
  const int K = a.K, KS = a.KS, C = a.C, J = a.J, B = a.B, nb = a.nb;
  const int BK = B * KS;
  const int SL = 2 * (BK + KS);
  const int tid = threadIdx.x;
  const int gid = tid / UPD_GROUP;         // 0: update group, 1: look-ahead group
  const int gt = tid - gid * UPD_GROUP;    // thread within the group
  const int lane = tid & 31, gw = gt >> 5;  // warp within the group
  const int grp = lane / UPD_LPR, gl = lane % UPD_LPR;  // UPD_RPW row groups of UPD_LPR lanes
  const int KS4 = KS >> 2;
  const int bar_id = 1 + gid;
  // shared memory carve-up: [sig KS] then per group: tab[max(2, nb)*KS] | part[GWARPS*KS] | ordS | prvS | segs
  const int tabn = (nb > 2 ? nb : 2) * KS;
  float* sig = smem;
  float* gbase = smem + KS + (size_t)gid * ((size_t)tabn + (size_t)UPD_GWARPS * KS + 2 * UPD_STAGE + ((J + 8) & ~3));
  float* tab = gbase;                          // update: Psum | lP ; look-ahead: Pprev[nb][KS]
  float* part = tab + tabn;                    // [GWARPS][KS]
  int* ordS = reinterpret_cast<int*>(part + UPD_GWARPS * KS);
  int* prvS = ordS + UPD_STAGE;
  int* segs = prvS + UPD_STAGE;                // [J + 1]
  constexpr int DEPTH_U = upd_depth_upd(NV), DEPTH_L = upd_depth_look(NV);
  const size_t group_floats = (size_t)tabn + (size_t)UPD_GWARPS * KS + 2 * UPD_STAGE + ((J + 8) & ~3);
  // per-warp cp.async ring [depth][rows][KS]: update-group warps first, then the look-ahead group's
  float* rowbuf = smem + KS + 2 * group_floats +
                  (gid == 0 ? (size_t)gw * (DEPTH_U * UPD_RPW * KS)
                            : (size_t)UPD_GWARPS * (DEPTH_U * UPD_RPW * KS) + (size_t)gw * (DEPTH_L * UPD_RPW * KS));
  __shared__ double sh_obj[2];

  for (int k = tid; k < KS; k += UPD_THREADS) sig[k] = (k < K) ? a.sigma[k] : 0.f;
  if (tid == 0) {
    sh_obj[0] = 0.0;
    sh_obj[1] = 0.0;
  }
  __syncthreads();

  float okd = 0.f, oent = 0.f;  // objective partials of the round in flight (group U only)
  auto tables_for = [&](int s) {
    SlotTables tv;
    const int par = (s - 1) & 1;
    tv.ringO = a.ring + (size_t)par * 2 * BK;
    tv.ringE = tv.ringO + BK;
    tv.prev = a.acc + (size_t)(s) * SL;      // slot(s-1) at index s
    tv.cur = a.acc + (size_t)(s + 1) * SL;   // slot(s)
    tv.BK = BK;
    tv.KS = KS;
    return tv;
  };

  // group-wide flush of per-lane column sums cs[NV][4] into dst_O[level][k] (+ dst_rs[k]) for tuple q
  auto flush = [&](float (&cs)[NV][4], int q, float* dst_O, float* dst_rs) {
#pragma unroll
    for (int v = 0; v < NV; ++v)
#pragma unroll
      for (int c = 0; c < 4; ++c) {
        float x = cs[v][c];
        x += __shfl_xor_sync(0xffffffffu, x, 16);
        cs[v][c] = 0.f;
        if (grp == 0) {
          int q4 = gl + UPD_LPR * v;
          if (q4 < KS4) part[gw * KS + q4 * 4 + c] = x;
        }
      }
    group_sync(bar_id);
    for (int k = gt; k < K; k += UPD_GROUP) {
      float t = 0.f;
#pragma unroll
      for (int w = 0; w < UPD_GWARPS; ++w) t += part[w * KS + k];
      atomicAdd(dst_rs + k, t);
      for (int c = 0; c < C; ++c) atomicAdd(dst_O + (size_t)a.tuple_levels[q * C + c] * KS + k, t);
    }
    group_sync(bar_id);
  };

  // ---- one block (round t, block j = step s) processed by the calling warp group ------------------
  // pre_wait: blocks until the step's inputs (counters) are complete; called after the plan data of the
  // step has been staged and the first row loads are in flight, right before the tables are derived
  auto process = [&](int s, auto mode_c, auto&& pre_wait) {
    constexpr int mode = decltype(mode_c)::value;
    constexpr int DEPTH = (mode == MODE_UPDATE) ? DEPTH_U : DEPTH_L;
    const int t = s / nb, j = s - t * nb;
    const bool single = a.ranges != nullptr;  // this CTA's rows of the block belong to ONE tuple
    int lo, hi, q = 0;
    if (single) {
      const int4 rg = __ldg(a.ranges + (size_t)s * gridDim.x + blockIdx.x);
      lo = rg.x;
      hi = rg.y;
      q = rg.z;
    } else {
      const int* ss = a.seg_start + (size_t)t * (nb * J + 1) + (size_t)j * J;
      for (int i = gt; i <= J; i += UPD_GROUP) segs[i] = ss[i];
      group_sync(bar_id);
      const int b0 = segs[0], b1 = segs[J];
      const int64_t blen = b1 - b0;
      lo = b0 + (int)((blen * blockIdx.x) / gridDim.x);
      hi = b0 + (int)((blen * (blockIdx.x + 1)) / gridDim.x);
    }
    if (lo >= hi) {
      pre_wait();
      return;
    }
    const int* order = a.order + (size_t)t * a.n;
    const int* prev_at = a.prev_at + (size_t)t * a.n;
    const bool writeR = (mode == MODE_UPDATE) && ((a.write_R_mask >> t) & 1u);
    float* dst_O;
    float* dst_rs;
    if (mode == MODE_UPDATE) {
      float* nslot = a.acc + (size_t)(s + 2) * SL;  // slot(s+1): add_s goes to its addprev part
      dst_O = nslot;
      dst_rs = nslot + BK;
    } else {
      float* slot = a.acc + (size_t)(s + 1) * SL;   // slot(s): rem_s
      dst_O = slot + BK + KS;
      dst_rs = dst_O + BK;
    }
    float cs[NV][4];
#pragma unroll
    for (int v = 0; v < NV; ++v)
#pragma unroll
      for (int c = 0; c < 4; ++c) cs[v][c] = 0.f;

    if (!single) {  // last q with segs[q] <= lo
      int l = 0, h = J;
      while (h - l > 1) {
        int m = (l + h) >> 1;
        if (segs[m] <= lo) l = m; else h = m;
      }
      q = l;
    }
    bool waited = false;
    for (int c0 = lo; c0 < hi; c0 += UPD_STAGE) {  // staged chunks of the CTA's range
      const int c1 = min(hi, c0 + UPD_STAGE);
      group_sync(bar_id);
      if (single && gt < C) segs[gt] = a.tuple_levels[q * C + gt];  // levels of this CTA's tuple (segs is free)
      for (int i = gt; i < c1 - c0; i += UPD_GROUP) {
        ordS[i] = order[c0 + i];
        if (mode == MODE_LOOK_U) prvS[i] = (t > 0) ? prev_at[c0 + i] : 0;
      }
      group_sync(bar_id);
      int p = c0;
      while (p < c1) {
        if (!single)
          while (segs[q + 1] <= p) ++q;  // skip empty segments
        const int run_end = single ? c1 : min(c1, segs[q + 1]);
        // --- start the cp.async row pipeline (DEPTH-1 batches), then derive this run's tables behind it
        const float* src = (mode == MODE_LOOK_R) ? a.R : a.U;
        auto issue = [&](int r0, int stage) {
          const int row = r0 + grp;
          if (row < run_end) {
            const int cell = ordS[row - c0];
            const float* gp = src + (size_t)cell * KS;
            const unsigned sp = (unsigned)__cvta_generic_to_shared(rowbuf + ((size_t)stage * UPD_RPW + grp) * KS);
#pragma unroll
            for (int v = 0; v < NV; ++v) {
              const int q4 = gl + UPD_LPR * v;
              if (q4 < KS4)
                asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(sp + q4 * 16), "l"(gp + q4 * 4) : "memory");
            }
          }
          asm volatile("cp.async.commit_group;" ::: "memory");
        };
        int r0 = p + gw * UPD_RPW;
#pragma unroll
        for (int i = 0; i < DEPTH - 1; ++i) issue(r0 + i * UPD_BATCH, i);
        if (!waited) {
          pre_wait();
          waited = true;
        }
        if constexpr (mode == MODE_UPDATE) {
          SlotTables tv = tables_for(s);
          for (int k = gt; k < KS; k += UPD_GROUP) {
            float v = 0.f;
            if (k < K)
              for (int c = 0; c < C; ++c) {
                float o, e, pp;
                derive(tv, a.Pr_b, a.theta, single ? segs[c] : a.tuple_levels[q * C + c], k, o, e, pp);
                v += pp;
              }
            tab[k] = v;                              // Psum
            tab[KS + k] = (k < K) ? fast_log(v) : 0.f;   // log Psum
          }
        } else if constexpr (mode == MODE_LOOK_U) {
          // previous-round penalty sums of tuple q for every block jp: tab[jp][k]
          const int sp_cur = s - 1;  // the step running right now in group U (its P is not saved yet)
          const int tp = t - 1;
          const int njp = (t == 0) ? 1 : nb;
          for (int idx = gt; idx < njp * KS; idx += UPD_GROUP) {
            const int jp = idx / KS, k = idx - jp * KS;
            float v = 0.f;
            if (k < K) {
              if (t == 0) {
                for (int c = 0; c < C; ++c) v += 1.f;  // R of the assignment step: plain softmax(U)
              } else {
                const int sp = tp * nb + jp;
                if (sp == sp_cur && !a.use_barrier) {  // per-step launches: P of the running step is not saved yet
                  SlotTables tv = tables_for(sp);
                  for (int c = 0; c < C; ++c) {
                    float o, e, pp;
                    derive(tv, a.Pr_b, a.theta, a.tuple_levels[q * C + c], k, o, e, pp);
                    v += pp;
                  }
                } else {
                  const float* Ps = a.Psave + ((size_t)(tp & 1) * nb + jp) * BK;
                  for (int c = 0; c < C; ++c) v += __ldcg(Ps + (size_t)(single ? segs[c] : a.tuple_levels[q * C + c]) * KS + k);
                }
              }
            }
            tab[idx] = v;
          }
        }
        group_sync(bar_id);
        // --- pipelined row loop: batches i+1 .. i+DEPTH-1 are in flight while batch i is reduced.
        // The loop is issue-bound: no branches (padding lanes / rows carry U_PAD -> exp = 0), the update
        // group's loop-invariant table rows live in registers.
        float4 pP[NV], pL[NV];
        bool slot_ok[NV];
#pragma unroll
        for (int v = 0; v < NV; ++v) {
          const int q4 = gl + UPD_LPR * v;
          slot_ok[v] = q4 < KS4;
          pP[v] = pL[v] = make_float4(0.f, 0.f, 0.f, 0.f);
          if constexpr (mode == MODE_UPDATE) {
            if (slot_ok[v]) {
              pP[v] = *reinterpret_cast<const float4*>(tab + q4 * 4);
              pL[v] = *reinterpret_cast<const float4*>(tab + KS + q4 * 4);
            }
          }
        }
        const bool sig_u = a.sigma_uniform != 0;
        for (int it = 0; r0 < run_end; r0 += UPD_BATCH, ++it) {
          issue(r0 + (DEPTH - 1) * UPD_BATCH, (it + DEPTH - 1) % DEPTH);
          asm volatile("cp.async.wait_group %0;" ::"n"(DEPTH - 1) : "memory");
          __syncwarp();
          const int row = r0 + grp;
          const bool valid = row < run_end;
          const int ridx = valid ? row - c0 : 0;
          const float* bp = rowbuf + ((size_t)(it % DEPTH) * UPD_RPW + grp) * KS;
          float4 ub[NV];
#pragma unroll
          for (int v = 0; v < NV; ++v) {
            const int q4 = gl + UPD_LPR * v;
            const float pad = (mode == MODE_LOOK_R) ? 0.f : U_PAD;
            ub[v] = make_float4(pad, pad, pad, pad);
            if (valid && slot_ok[v]) ub[v] = *reinterpret_cast<const float4*>(bp + q4 * 4);
          }
          if constexpr (mode == MODE_LOOK_R) {
#pragma unroll
            for (int v = 0; v < NV; ++v) {
              cs[v][0] += ub[v].x;
              cs[v][1] += ub[v].y;
              cs[v][2] += ub[v].z;
              cs[v][3] += ub[v].w;
            }
          } else {
            // exp through ex2.approx (2 ulp) and one reciprocal per row (IEEE expf / divides cost 3x)
            float ssum = 0.f, Aacc = 0.f, Bacc = 0.f, Sacc = 0.f;
            const float* pw = tab + (size_t)((mode == MODE_LOOK_U) ? prvS[ridx] : 0) * KS;
#pragma unroll
            for (int v = 0; v < NV; ++v) {  // ub[v] <- exp(u) * Psum (the un-normalised R, >= 0)
              const int q4 = gl + UPD_LPR * v;
              float4 p4 = pP[v];
              if constexpr (mode == MODE_LOOK_U) {
                p4 = make_float4(0.f, 0.f, 0.f, 0.f);
                if (slot_ok[v]) p4 = *reinterpret_cast<const float4*>(pw + q4 * 4);
              }
              const float4 u4 = ub[v];
              ub[v].x = fast_exp(u4.x) * p4.x;
              ub[v].y = fast_exp(u4.y) * p4.y;
              ub[v].z = fast_exp(u4.z) * p4.z;
              ub[v].w = fast_exp(u4.w) * p4.w;
              if constexpr (mode == MODE_UPDATE) {
                const float4 l4 = pL[v];
                if (sig_u) {
                  Aacc = fmaf(ub[v].x, u4.x, Aacc); Bacc = fmaf(ub[v].x, l4.x, Bacc);
                  Aacc = fmaf(ub[v].y, u4.y, Aacc); Bacc = fmaf(ub[v].y, l4.y, Bacc);
                  Aacc = fmaf(ub[v].z, u4.z, Aacc); Bacc = fmaf(ub[v].z, l4.z, Bacc);
                  Aacc = fmaf(ub[v].w, u4.w, Aacc); Bacc = fmaf(ub[v].w, l4.w, Bacc);
                } else {
                  const float4 s4 = slot_ok[v] ? *reinterpret_cast<const float4*>(sig + q4 * 4) : make_float4(0.f, 0.f, 0.f, 0.f);
                  float tt;
                  tt = s4.x * ub[v].x; Aacc = fmaf(tt, u4.x, Aacc); Bacc = fmaf(tt, l4.x, Bacc); Sacc += tt;
                  tt = s4.y * ub[v].y; Aacc = fmaf(tt, u4.y, Aacc); Bacc = fmaf(tt, l4.y, Bacc); Sacc += tt;
                  tt = s4.z * ub[v].z; Aacc = fmaf(tt, u4.z, Aacc); Bacc = fmaf(tt, l4.z, Bacc); Sacc += tt;
                  tt = s4.w * ub[v].w; Aacc = fmaf(tt, u4.w, Aacc); Bacc = fmaf(tt, l4.w, Bacc); Sacc += tt;
                }
              }
              ssum += (ub[v].x + ub[v].y) + (ub[v].z + ub[v].w);
            }
            ssum += __shfl_xor_sync(0xffffffffu, ssum, 1);
            ssum += __shfl_xor_sync(0xffffffffu, ssum, 2);
            ssum += __shfl_xor_sync(0xffffffffu, ssum, 4);
            ssum += __shfl_xor_sync(0xffffffffu, ssum, 8);
            const float sdiv = (ssum == 0.f) ? 1.f : ssum;  // arma::normalise(.., 1, 0): zero norm divides by 1
            const float inv = fast_rcp(sdiv);
            float4* rp = reinterpret_cast<float4*>(a.R + (size_t)ordS[ridx] * KS);
#pragma unroll
            for (int v = 0; v < NV; ++v) {
              const int q4 = gl + UPD_LPR * v;
              float4 r;
              r.x = ub[v].x * inv;
              r.y = ub[v].y * inv;
              r.z = ub[v].z * inv;
              r.w = ub[v].w * inv;
              cs[v][0] += r.x;
              cs[v][1] += r.y;
              cs[v][2] += r.z;
              cs[v][3] += r.w;
              if (writeR && valid && slot_ok[v]) rp[q4] = r;
            }
            if constexpr (mode == MODE_UPDATE) {
              // sum_k R dist = -sum sigma R U ;  sum_k sigma R log R = sum sigma R (U + log Psum - log s)
              const float ls = fast_log(sdiv);
              if (sig_u) {
                // per lane: Sacc would be this lane's share of ssum; use the row total once (lane gl == 0)
                const float srow = (gl == 0) ? ssum : 0.f;
                okd -= a.sigma0 * inv * Aacc;
                oent += a.sigma0 * inv * (Aacc + Bacc - ls * srow);
              } else {
                okd -= inv * Aacc;
                oent += inv * (Aacc + Bacc - ls * Sacc);
              }
            }
          }
          __syncwarp();  // the stage is refilled by the next iteration's issue
        }
        asm volatile("cp.async.wait_group 0;" ::: "memory");
        flush(cs, q, dst_O, dst_rs);
        p = run_end;
      }
    }
  };

  // ---- owners: materialise O_s, E_s (ring), the end-of-round tables and save P_s (group U threads) ----
  auto owners = [&](int s) {
    const int t = s / nb, j = s - t * nb;
    SlotTables tv = tables_for(s);
    float* outO = a.ring + (size_t)(s & 1) * 2 * BK;
    float* outE = outO + BK;
    float* Ps = a.Psave + ((size_t)(t & 1) * nb + j) * BK;
    for (int idx = blockIdx.x * UPD_GROUP + gt; idx < BK; idx += gridDim.x * UPD_GROUP) {
      const int b = idx / KS, k = idx - b * KS;
      float o = 0.f, e = 0.f, pp = 0.f;
      if (k < K) derive(tv, a.Pr_b, a.theta, b, k, o, e, pp);
      outO[idx] = o;
      outE[idx] = e;
      Ps[idx] = pp;
      if (j == 0 && t > 0) {
        float* oe = a.OEend + (size_t)(t - 1) * 2 * BK;
        oe[idx] = o;
        oe[BK + idx] = e;
      }
    }
  };
  auto flush_objective = [&](int t) {  // group U
    okd = warp_sum(okd);
    oent = warp_sum(oent);
    if (lane == 0) {
      atomicAdd(&sh_obj[0], (double)okd);
      atomicAdd(&sh_obj[1], (double)oent);
    }
    group_sync(bar_id);
    if (gt == 0) {
      atomicAdd(a.obj + 2 * t + 0, sh_obj[0]);
      atomicAdd(a.obj + 2 * t + 1, sh_obj[1]);
      sh_obj[0] = 0.0;
      sh_obj[1] = 0.0;
    }
    group_sync(bar_id);
    okd = 0.f;
    oent = 0.f;
  };

  // ---- completion counters (cooperative launch only): cntU[s], cntL[s] = #CTAs whose group finished step s
  const int S_total = a.T * nb;
  unsigned* cntU = a.bar + 1;                  // index s + 1 is folded in: cntU[s] for s >= -1
  unsigned* cntL = a.bar + (S_total + 2) + 1;
  auto signal = [&](unsigned* c) {
    group_sync(bar_id);
    if (gt == 0) {
      __threadfence();
      asm volatile("red.release.gpu.global.add.u32 [%0], 1;" ::"l"(c) : "memory");
    }
  };
  auto wait_for = [&](const unsigned* c) {
    if (gt == 0) {
      while (ld_acquire_u32(c) < gridDim.x) __nanosleep(20);
      __threadfence();
    }
    group_sync(bar_id);
  };
  auto no_wait = [&]() {};
  if (gid == 0) {
    // ---------------- update group: the critical path ----------------
    for (int s = a.s_begin; s < a.s_end; ++s) {
      auto waits = [&]() {
        if (a.use_barrier) {
          if (s > a.s_begin) wait_for(cntU + s - 1);                 // add_{s-1}, ring, Psave of step s-1
          if (s > a.s_begin || a.prologue) wait_for(cntL + s);       // rem_s
        }
        owners(s);
      };
      process(s, std::integral_constant<int, MODE_UPDATE>(), waits);
      if ((s + 1) % nb == 0) flush_objective(s / nb);
      if (a.use_barrier) signal(cntU + s);
    }
    if (a.s_end % nb != 0 && a.s_end > a.s_begin) flush_objective((a.s_end - 1) / nb);  // partial round
  } else {
    // ---------------- look-ahead group: streams ahead of the update group ----------------
    const int first = a.prologue ? a.s_begin : a.s_begin + 1;
    const int last = (a.s_end < S_total) ? a.s_end : S_total - 1;   // look-ahead targets: first .. last
    for (int s = first; s <= last; ++s) {
      auto waits = [&]() {
        if (a.use_barrier) {
          const int t = s / nb;
          // tables of the previous round must all be saved (its last step's owners signal through cntU)
          int need = (t > 0) ? t * nb - 1 : -1;
          const int bound = s - UPD_RUNAHEAD;                           // L2 footprint: stay <= UPD_RUNAHEAD steps ahead
          if (bound > need) need = bound;
          if (need >= a.s_begin) wait_for(cntU + need);
        }
      };
      if (s < nb && a.first_round_from_R)
        process(s, std::integral_constant<int, MODE_LOOK_R>(), waits);
      else
        process(s, std::integral_constant<int, MODE_LOOK_U>(), waits);
      if (a.use_barrier) signal(cntL + s);
    }
  }
}

// After the last executed step S: O = O_S, E = E_S into the handle's tables (and the objective tables).
__global__ void k_two_pass_finalize(TwoPassArgs a, int S, float* __restrict__ O, float* __restrict__ E) {
  const int KS = a.KS, BK = a.B * KS, SL = 2 * (BK + KS);
  const float* ringO = a.ring + (size_t)((S - 1) & 1) * 2 * BK;
  const float* ringE = ringO + BK;
  const float* prev = a.acc + (size_t)(S)*SL;
  const float* cur = a.acc + (size_t)(S + 1) * SL;
  for (int idx = blockIdx.x * blockDim.x + threadIdx.x; idx < BK; idx += gridDim.x * blockDim.x) {
    const int b = idx / KS, k = idx - b * KS;
    float o = 0.f, e = 0.f;
    if (k < a.K) {
      // same arithmetic as derive() without the removal of step S (which never runs)
      const float prb = a.Pr_b[b];
      const float* prev_rem_O = prev + BK + KS;
      const float* prev_rem_rs = prev_rem_O + BK;
      o = (ringO[idx] - prev_rem_O[idx]) + cur[idx];
      e = (ringE[idx] - prev_rem_rs[k] * prb) + cur[BK + k] * prb;
    }
    O[idx] = o;
    E[idx] = e;
  }
}

}  // namespace hb
