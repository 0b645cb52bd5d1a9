// update_slots.cuh — the step protocol the two persistent update_R kernels (update_two_pass.cuh,
// update_single_pass.cuh) share: accumulator slots, the derivation of a step's K x B tables from them, the
// completion counters' acquire load, and the peer-memory words that carry a slot's add half between GPUs.
//
// Per-step accumulators of one cluster_cpp call live in `acc`: slot(s) = [add_{s-1} | rem_s], s = -1 .. S, at
// index s + 1, each [add_O B*KS | add_rs KS | rem_O B*KS | rem_rs KS], zeroed by the host before the first
// launch.  Derivation (reference order of operations):
//   O_s = (O_{s-1} - rem_{s-1}) + add_{s-1}        E likewise with row sums * Pr_b
//   P_s = ((2 (E_s - rs_rem_s Pr_b) + 1) / ((O_s - rem_s) + (E_s - rs_rem_s Pr_b) + 1)) ^ theta
#pragma once
#include "common.cuh"

namespace hb {

__device__ __forceinline__ unsigned ld_acquire_u32(const unsigned* p) {
  unsigned v;
  asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}

// Sharded cells on one node (one process per GPU): the per-step sums cross GPUs through peer memory instead of a
// collective per block step.  Every rank owns an exchange area that all ranks of the node have mapped (CUDA IPC
// over NVLink):  inbox[slot][src][XH]  (XH = B KS + KS values: the add half of an accumulator slot) and the rank's
// remT tables.  The CTA that completes the LOCAL add half of a slot copies it into entry src = rank of every
// rank's inbox; readers add the entries in rank order, so every rank derives bit-identical tables.  The next
// round's removal sums are read from the peers' remT directly when a round is folded.
constexpr int XCH_MAXWORLD = 8;
struct PeerXch {
  int world = 1, rank = 0;
  unsigned epoch = 0;
  int XH = 0;
  uint2* inbox = nullptr;       // local area: [slot][src][XH] of (value bits, epoch)
  uint2* peer_inbox[XCH_MAXWORLD] = {};
  float* peer_remT[XCH_MAXWORLD] = {};  // every rank's remT (own entry = local pointer)
};

// Low-latency exchange words: every value travels with the epoch of the running cluster_cpp call in ONE 8-byte
// store (single-copy atomic), so a reader needs neither a flag nor a fence: it polls the word it wants until the
// epoch matches.  One NVLink one-way latency per block step instead of data + system fence + flag.
__device__ __forceinline__ uint2 xch_ld(const uint2* p) {
  uint2 v;
  asm volatile("ld.relaxed.sys.global.v2.u32 {%0,%1}, [%2];" : "=r"(v.x), "=r"(v.y) : "l"(p) : "memory");
  return v;
}
// two consecutive words in one 16-byte store (p 16-byte aligned): each 64-bit element is single-copy atomic and
// carries its own epoch, so the pair needs no atomicity as a whole — half the packets on the fabric
__device__ __forceinline__ void xch_st2(uint2* p, float v0, float v1, unsigned epoch) {
  const unsigned long long w0 = ((unsigned long long)epoch << 32) | __float_as_uint(v0);
  const unsigned long long w1 = ((unsigned long long)epoch << 32) | __float_as_uint(v1);
  asm volatile("st.relaxed.sys.global.v2.u64 [%0], {%1,%2};" ::"l"(p), "l"(w0), "l"(w1) : "memory");
}
// sum over the ranks' entries of element `off` of the add half of accumulator slot index `sl`, in rank order
// (waits for entries that have not arrived yet)
__device__ __forceinline__ float xch_sum(const PeerXch& x, int sl, int off) {
  const uint2* q = x.inbox + ((size_t)sl * x.world) * x.XH + off;
  float t = 0.f;
  for (int r = 0; r < x.world; ++r) {
    uint2 v = xch_ld(q + (size_t)r * x.XH);
    while (v.y != x.epoch) {
      __nanosleep(20);
      v = xch_ld(q + (size_t)r * x.XH);
    }
    t += __uint_as_float(v.x);
  }
  return t;
}

// ((2E+1)/(O+E+1))^theta (harmony_pow, utils.cpp:84-90) as ex2(theta * lg2(x)): the tables sit on the critical
// path of every block step and powf costs ~100 instructions; x > 0 here, theta = 0 gives exactly 1.
__device__ __forceinline__ float penalty_pow(float o_eff, float e_eff, float th) {
  const float x = ((2.f * e_eff) + 1.f) / (o_eff + e_eff + 1.f);
  float l, y;
  asm("lg2.approx.ftz.f32 %0, %1;" : "=f"(l) : "f"(x));
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(th * l));
  return y;
}

struct SlotTables {
  const float* ringO;   // O_{s-1}
  const float* ringE;
  const float* prev;    // slot(s-1)
  const float* cur;     // slot(s)
  int BK, KS;
};
// O_s, E_s and P_s of element (b, k); every input was completed before the counter this CTA waited for -> L2 loads
// (.cg).  xs >= 0: sharded cells, the add half of slot index xs is the sum of the ranks' inbox entries (xs < 0: none)
__device__ __forceinline__ void derive(const SlotTables& tv, const float* Pr_b, const float* theta, int b, int k, float& o,
                                       float& e, float& p, const PeerXch* x = nullptr, int xs = -1) {
  const int idx = b * tv.KS + k;
  const float prb = __ldg(Pr_b + b);
  const float* prev_rem_O = tv.prev + tv.BK + tv.KS;
  const float* prev_rem_rs = prev_rem_O + tv.BK;
  const float* cur_add_O = tv.cur;
  const float* cur_add_rs = tv.cur + tv.BK;
  const float* cur_rem_O = tv.cur + tv.BK + tv.KS;
  const float* cur_rem_rs = cur_rem_O + tv.BK;
  float add_o, add_rs;
  if (x) {
    add_o = (xs >= 0) ? xch_sum(*x, xs, idx) : 0.f;
    add_rs = (xs >= 0) ? xch_sum(*x, xs, tv.BK + k) : 0.f;
  } else {
    add_o = __ldcg(cur_add_O + idx);
    add_rs = __ldcg(cur_add_rs + k);
  }
  o = (__ldcg(tv.ringO + idx) - __ldcg(prev_rem_O + idx)) + add_o;
  e = (__ldcg(tv.ringE + idx) - __ldcg(prev_rem_rs + k) * prb) + add_rs * prb;
  const float e_eff = e - __ldcg(cur_rem_rs + k) * prb;
  const float o_eff = o - __ldcg(cur_rem_O + idx);
  p = penalty_pow(o_eff, e_eff, __ldg(theta + b));
}

}  // namespace hb
