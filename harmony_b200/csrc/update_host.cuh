// update_host.cuh — the update_R launchers (per step, two-pass, single-pass) and the state they keep per cluster_cpp
// call.  Included by harmony_b200.cu after tuples.cuh.
#pragma once

namespace {

// exchange area of the persistent update kernel for sharded cells (see setup_peer_exchange)
struct XchArea {
  int device = 0, world = 0, rank = 0;
  size_t slots = 0, XH = 0, remT_floats = 0;
  float* base = nullptr;     // [inbox: slots * world * XH floats | flags: slots * world words | remT: remT_floats]
  void* peer[XCH_MAXWORLD] = {};
  unsigned epoch = 0;
  bool leased = false;
};

struct UpdateState {
  size_t BK = 0, XH = 0;  // floats of a K x B table [B][KS], and of half a slot (a table and its row sums)
  int rounds = 0;         // the round-sized buffers hold calls of up to this many rounds
  DevBuf<float> acc, P;   // per-step path: its two slots, the P table of a step
  DevBuf<float> ring, acc2, Psave, OEend;  // persistent kernels: table ring, slots, P per block, tables per round
  DevBuf<double> obj2;    // objective sums per round
  DevBuf<unsigned> bar;   // step counters
  DevBuf<float> remT;     // [2][nb][J][KS] next round's removal sums per (block, tuple)
  DevBuf<float> remS;     // [nb][J][KS] sharded cells: the ranks' remT of one round, summed
  DevBuf<int> lvl_ptr, lvl_tup;  // CSR level -> tuples (+ one trailing word: B_vec[0])
  int ring_rows = 0;      // rows of a warp's private ring in the single-pass update kernel
  bool use_xch = false;   // sharded cells: block steps exchanged through peer memory (one cooperative launch per call)
  PeerXch xch{};
  XchArea* xarea = nullptr;  // leased exchange area (process-wide pool, see setup_peer_exchange)

  // A slot is [add_O | add_rs | rem_O | rem_rs] (update_slots.cuh): slot s of the persistent kernels (0 .. T nb + 1),
  // or slot j of the per-step path, which takes its two slots in turn
  size_t slot_floats() const { return 2 * XH; }
  float* slot(size_t s) const { return acc2.p + s * slot_floats(); }
  float* step_slot(int j) const { return acc.p + (size_t)(j & 1) * slot_floats(); }
  float* rem_half(float* slot) const { return slot + XH; }
  // ring[1] (= "O_{-1}"): the tables a call starts from
  float* seed_O() const { return ring.p + 2 * BK; }
  float* seed_E() const { return ring.p + 3 * BK; }
};

// ---- peer-memory exchange area of the persistent update kernel (sharded cells, one node) ----------------
// Areas live for the life of the process, like the communicators: another rank may still be writing into an
// area when its owner drops the handle, and unmapping needs a collective that a destructor cannot afford.  A
// handle leases an area; areas are created collectively, so area i here is paired with area i of every rank.
constexpr int XCH_MAX_AREAS = 16;
std::vector<XchArea*> g_xch_areas;

void release_peer_exchange(hb_handle* h) {
  UpdateState& u = *h->upd;
  if (u.xarea) {
    u.xarea->epoch = u.xch.epoch;  // the next lessee continues the epoch sequence
    u.xarea->leased = false;
    u.xarea = nullptr;
  }
  u.use_xch = false;
}
// layout of an area (floats): inbox [slots][world][XH] of 8-byte (value, epoch) words | remT [2][nb][J][KS]
uint2* xch_inbox(const XchArea* a, void* base) { return reinterpret_cast<uint2*>(base); }
float* xch_remT(const XchArea* a, void* base) { return reinterpret_cast<float*>(base) + 2 * a->slots * a->world * a->XH; }
// Collective over the handle's communicator.  Leases an area all ranks have free, or creates a new one:
// allocates this rank's part, exchanges the IPC handles and maps the other ranks' parts.  If any rank cannot
// map a peer the exchange stays off on all ranks (the update then runs one launch + all-reduce per block step).
int setup_peer_exchange(hb_handle* h, int Tplan) {
  UpdateState& u = *h->upd;
  const int W = h->world;
  const size_t XH = u.XH;
  const size_t slots = (size_t)Tplan * h->nb + 2;
  const size_t remT_floats = 2 * (size_t)h->nb * h->J * h->KS;
  release_peer_exchange(h);
  // 1. agree on a reusable area: free here AND on every other rank, same shape
  int64_t freev[XCH_MAX_AREAS + 2];
  for (int i = 0; i < XCH_MAX_AREAS; ++i) {
    const XchArea* a = i < (int)g_xch_areas.size() ? g_xch_areas[i] : nullptr;
    freev[i] = (a && !a->leased && a->device == h->device && a->world == W && a->rank == h->rank && a->slots == slots &&
                a->XH == XH && a->remT_floats == remT_floats) ? 1 : 0;
  }
  freev[XCH_MAX_AREAS] = (int64_t)g_xch_areas.size();       // min over ranks = smallest pool ...
  freev[XCH_MAX_AREAS + 1] = -(int64_t)g_xch_areas.size();  // ... and -(largest pool): they must agree
  DevBuf<int64_t> dv;
  CK(dv.alloc(XCH_MAX_AREAS + 2));
  CK(cudaMemcpyAsync(dv.p, freev, sizeof(freev), cudaMemcpyHostToDevice, h->stream));
  CKN(g_nccl.AllReduce(dv.p, dv.p, XCH_MAX_AREAS + 2, ncclInt64, ncclMin, h->comm, h->stream));
  CK(cudaMemcpyAsync(freev, dv.p, sizeof(freev), cudaMemcpyDeviceToHost, h->stream));
  CK(cudaStreamSynchronize(h->stream));
  XchArea* area = nullptr;
  for (int i = 0; i < XCH_MAX_AREAS && !area; ++i)
    if (freev[i] == 1) area = g_xch_areas[i];
  if (!area) {
    // every rank sees the same reduced values, so every rank takes the same branch here
    if (freev[XCH_MAX_AREAS] != -freev[XCH_MAX_AREAS + 1] || freev[XCH_MAX_AREAS] >= XCH_MAX_AREAS) return 0;  // out of step / pool full
    // 2. create a new area (collective)
    XchArea made{h->device, W, h->rank, slots, XH, remT_floats};
    const size_t total = (size_t)(xch_remT(&made, nullptr) - (float*)nullptr) + remT_floats;
    CK(cudaMalloc((void**)&made.base, sizeof(float) * total));
    CK(cudaMemsetAsync(made.base, 0, sizeof(float) * total, h->stream));
    cudaIpcMemHandle_t mine;
    CK(cudaIpcGetMemHandle(&mine, made.base));
    DevBuf<char> ds, dr;
    CK(ds.alloc(sizeof(mine)));
    CK(dr.alloc(sizeof(mine) * W));
    CK(cudaMemcpyAsync(ds.p, &mine, sizeof(mine), cudaMemcpyHostToDevice, h->stream));
    CKN(g_nccl.AllGather(ds.p, dr.p, sizeof(mine), ncclChar, h->comm, h->stream));
    std::vector<cudaIpcMemHandle_t> all(W);
    CK(cudaMemcpyAsync(all.data(), dr.p, sizeof(mine) * W, cudaMemcpyDeviceToHost, h->stream));
    CK(cudaStreamSynchronize(h->stream));
    area = new XchArea(made);
    int64_t ok = 1;
    for (int r = 0; r < W; ++r) {
      if (r == h->rank) continue;
      if (cudaIpcOpenMemHandle(&area->peer[r], all[r], cudaIpcMemLazyEnablePeerAccess) != cudaSuccess) {
        cudaGetLastError();
        area->peer[r] = nullptr;
        ok = 0;
      }
    }
    CK(cudaMemcpyAsync(dv.p, &ok, sizeof(ok), cudaMemcpyHostToDevice, h->stream));
    CKN(g_nccl.AllReduce(dv.p, dv.p, 1, ncclInt64, ncclMin, h->comm, h->stream));
    CK(cudaMemcpyAsync(&ok, dv.p, sizeof(ok), cudaMemcpyDeviceToHost, h->stream));
    CK(cudaStreamSynchronize(h->stream));
    area->leased = !ok;            // an unusable area keeps its index (the ranks stay in step) but is never leased
    g_xch_areas.push_back(area);
    if (!ok) {
      h->warnings.push_back("peer-memory exchange unavailable (CUDA IPC mapping failed); using per-step all-reduce");
      return 0;
    }
  }
  area->leased = true;
  u.xarea = area;
  PeerXch& x = u.xch;
  x.world = W;
  x.rank = h->rank;
  x.epoch = area->epoch;
  x.XH = (int)XH;
  for (int r = 0; r < W; ++r) {
    void* b = (r == h->rank) ? (void*)area->base : area->peer[r];
    x.peer_inbox[r] = xch_inbox(area, b);
    x.peer_remT[r] = xch_remT(area, b);
  }
  x.inbox = x.peer_inbox[h->rank];
  u.use_xch = true;
  return 0;
}
float* remT_ptr(hb_handle* h) { return h->upd->use_xch ? h->upd->xch.peer_remT[h->rank] : h->upd->remT.p; }

// The update state for calls of up to T rounds: everything on the first call (hb_setup), afterwards the buffers sized
// by the rounds of a call.  Growing sets the exchange area up again, a collective: every rank grows its plan in the
// same call.
int update_reserve(hb_handle* h, int T) {
  UpdateState& u = *h->upd;
  const bool first = u.rounds == 0;
  u.rounds = T;
  u.BK = (size_t)h->B * h->KS;
  u.XH = u.BK + h->KS;
  if (first) {
    u.ring_rows = sp_ring_rows(h->KS, SMEM_LIMIT);
    CK(u.acc.alloc(2 * u.slot_floats()));
    CK(u.P.alloc(u.BK));
  }
  if (h->paths.update == UpdatePath::PerStep) return 0;
  const size_t slots = (size_t)T * h->nb + 2;
  CK(u.acc2.alloc(u.slot_floats() * slots));
  CK(u.OEend.alloc((size_t)T * 2 * u.BK));
  CK(u.obj2.alloc(2 * (size_t)T));
  CK(u.bar.alloc(2 * slots));
  if (!first) return u.use_xch ? setup_peer_exchange(h, T) : 0;
  const bool single_pass = h->paths.update == UpdatePath::SinglePass;
  CK(u.ring.alloc(4 * u.BK));
  CK(u.Psave.alloc(single_pass ? 1 : 2 * (size_t)h->nb * u.BK));
  if (single_pass) CK(u.remT.alloc(2 * (size_t)h->nb * h->J * h->KS));
  if (single_pass && h->world > 1) CK(u.remS.alloc((size_t)h->nb * h->J * h->KS));
  if (single_pass && h->world > 1 && h->world <= XCH_MAXWORLD && !(h->kernel_set & HB_KS_NO_PEER_EXCHANGE))
    TRY(setup_peer_exchange(h, T));
  CK(cudaMemsetAsync(u.Psave.p, 0, sizeof(float) * u.Psave.n, h->stream));
  CK(cudaMemsetAsync(u.ring.p, 0, sizeof(float) * 4 * u.BK, h->stream));
  return 0;
}

// Starts a call of T rounds on a persistent path: zeroes the slots, objective sums and step counters, runs
// cold_start() (the plan-order assignment of a call that runs one: it fills the removal halves of slots 1 .. nb, and
// O and E), and seeds ring[1] with the tables the call starts from.
template <typename F>
int update_begin(hb_handle* h, int T, F&& cold_start) {
  if (T == 0) return 0;
  UpdateState& u = *h->upd;
  const size_t slots = (size_t)T * h->nb + 2;
  CK(cudaMemsetAsync(u.acc2.p, 0, sizeof(float) * u.slot_floats() * slots, h->stream));
  CK(cudaMemsetAsync(u.obj2.p, 0, sizeof(double) * 2 * (size_t)T, h->stream));
  CK(cudaMemsetAsync(u.bar.p, 0, sizeof(unsigned) * 2 * slots, h->stream));
  if (h->paths.update == UpdatePath::SinglePass) CK(cudaMemsetAsync(remT_ptr(h), 0, sizeof(float) * 2 * (size_t)h->nb * h->J * h->KS, h->stream));
  if (u.use_xch) u.xch.epoch++;  // flags of earlier calls no longer match
  TRY(cold_start());
  CK(cudaMemcpyAsync(u.seed_O(), h->O.p, sizeof(float) * u.BK, cudaMemcpyDeviceToDevice, h->stream));
  CK(cudaMemcpyAsync(u.seed_E(), h->E.p, sizeof(float) * u.BK, cudaMemcpyDeviceToDevice, h->stream));
  return 0;
}

// ---- per-step path: one update_R sweep (harmony.cpp:269-342), three launches per block step ---------------
int run_update_per_step(hb_handle* h) {
  RegionScope rs(h, "update_R");
  const UpdateState& u = *h->upd;
  const int K = h->K, B = h->B, nb = h->nb, KS = h->KS;
  const int KP = (K + 63) & ~63;
  const size_t BK = u.BK, slot = u.slot_floats();
  CK(cudaMemsetAsync(u.acc.p, 0, sizeof(float) * 2 * slot, h->stream));
  const PlanRound0 r = plan_round0(h, 0);  // the one round the per-step path plans
  StepArgs a;
  a.U = h->U.p;
  a.R = h->R.p;
  a.order = r.order;
  a.seg_start = r.seg_start;
  a.tile_base = r.tile_base;
  a.tuple_levels = h->tuple_levels.p;
  a.sigma = h->sigma.p;
  a.P = u.P.p;
  a.obj_acc = h->obj_acc.p;
  a.J = h->J;
  a.K = K;
  a.C = h->C;
  a.KP = KP;
  a.KS = KS;
  const int grid = std::max(1, (int)std::min<int64_t>((h->n / std::max(1, nb)) / TM + h->J + 8, (int64_t)h->num_sms * 8));
  const size_t sm_col = sizeof(float) * (size_t)NWARP * KP;
  const size_t sm_upd = sizeof(float) * ((size_t)NWARP * KP + 3 * (size_t)KP);
  return dispatch<1, 2, 4, 8, 16, 32>(h, kq_for(K), kUnsupportedK, [&](auto kq) -> int {
    constexpr int KQ = decltype(kq)::value;
    for (int j = 0; j <= nb; ++j) {
      float* sl = u.step_slot(j);  // slot j = [add_{j-1} | rem_j]
      float* rem = u.rem_half(sl);
      if (j < nb) {
        a.blk = j;
        a.acc_O = rem;
        a.acc_rs = rem + BK;
        RegionScope r1(h, "k_block_colsum");
        k_block_colsum<KQ><<<grid, ROW_THREADS, sm_col, h->stream>>>(a);
        CKL();
      }
      TRY(allreduce_f(h, sl, slot));
      {
        RegionScope r2(h, "k_step_prepare");
        k_step_prepare<<<(B * KS + 255) / 256, 256, 0, h->stream>>>(h->O.p, h->E.p, sl, sl + BK, rem, rem + BK, h->Pr_b.p,
                                                                     h->theta.p, (j < nb) ? u.P.p : nullptr, B, K, KS);
        CKL();
      }
      CK(cudaMemsetAsync(sl, 0, sizeof(float) * slot, h->stream));
      if (j < nb) {
        float* nx = u.step_slot(j + 1);  // add_j goes to slot j+1
        a.acc_O = nx;
        a.acc_rs = nx + BK;
        RegionScope r3(h, "k_block_update");
        k_block_update<KQ><<<grid, ROW_THREADS, sm_upd, h->stream>>>(a);
        CKL();
      }
    }
    return 0;
  });
}

// ---- persistent update kernels over rounds [t0, t1) of this cluster_cpp call ---------------------------
// the arguments both persistent kernels take (TwoPassArgs, SinglePassArgs) for a call of T rounds from round 0 r
template <typename A>
A persistent_args(hb_handle* h, int T, const PlanRound0& r) {
  const UpdateState& u = *h->upd;
  A a;
  a.U = h->U.p;
  a.R = h->R.p;
  a.order = r.order;
  a.ranges = r.ranges;
  a.tuple_levels = h->tuple_levels.p;
  a.sigma = h->sigma.p;
  a.theta = h->theta.p;
  a.Pr_b = h->Pr_b.p;
  a.ring = u.ring.p;
  a.acc = u.acc2.p;
  a.OEend = u.OEend.p;
  a.obj = u.obj2.p;
  a.bar = u.bar.p;
  a.n = h->n;
  a.K = h->K;
  a.KS = h->KS;
  a.C = h->C;
  a.J = h->J;
  a.B = h->B;
  a.nb = h->nb;
  a.T = T;
  a.sigma_uniform = h->sigma_uniform ? 1 : 0;
  a.sigma0 = h->sigma0;
  return a;
}
int launch_two_pass(hb_handle* h, TwoPassArgs a, bool cooperative) {
  const size_t smem = two_pass_smem_bytes(h->KS, h->nb, h->J);
  a.use_barrier = cooperative ? 1 : 0;
  return dispatch<1, 2, 4>(h, two_pass_nv(h->KS), kUnsupportedUpdateK, [&](auto nvc) -> int {
    return launch_coop(h, k_update_two_pass<decltype(nvc)::value>, cooperative, h->coop_grid, UPD_THREADS, smem, a);
  });
}
int launch_single_pass(hb_handle* h, SinglePassArgs a, bool cooperative) {
  a.coop = cooperative ? 1 : 0;
  SinglePassLaunch lp;
  lp.a = a;
  if (h->upd->use_xch) lp.x = h->upd->xch;
  return dispatch<1, 2>(h, sp_nv(h->KS), kUnsupportedUpdateK, [&](auto nvc) {
    constexpr int NV = decltype(nvc)::value;
    const size_t smem = sp_smem_bytes(NV, a.ring_rows, a.KS);
    // sigma_uniform, the default: scalar sigma (objective terms simplify)
    return launch_coop(h, h->sigma_uniform ? k_update_single_pass<NV, true> : k_update_single_pass<NV, false>, cooperative,
                       h->coop_grid, SP_THREADS, smem, lp);
  });
}
// compute_objective() of every round in [t0, t1) (harmony.cpp:248) from the kernels' per-round sums and tables
int push_round_objectives(hb_handle* h, int t0, int t1) {
  const UpdateState& u = *h->upd;
  for (int t = t0; t < t1; ++t) {
    const float* O = (t == t1 - 1) ? h->O.p : u.OEend.p + (size_t)t * 2 * u.BK;
    const float* E = (t == t1 - 1) ? h->E.p : u.OEend.p + (size_t)t * 2 * u.BK + u.BK;
    TRY(push_objective_from(h, O, E, u.obj2.p + 2 * (size_t)t));
  }
  return 0;
}
// single-pass kernel (update_single_pass.cuh), rounds [t0, t1)
int run_update_single_pass(hb_handle* h, int T, int t0, int t1, bool rem_ready) {
  RegionScope rs(h, "update_R");
  const UpdateState& u = *h->upd;
  const int nb = h->nb;
  const PlanRound0 r = plan_round0(h, h->plan->set);
  SinglePassArgs a = persistent_args<SinglePassArgs>(h, T, r);
  a.next_at = r.next_at;
  a.lvl_ptr = u.lvl_ptr.p;
  a.lvl_tup = u.lvl_tup.p;
  a.lvl_first1 = u.lvl_ptr.p + h->B + 1;
  a.remT = remT_ptr(h);
  a.remS = u.remS.p;
  a.s_begin = a.s_end = 0;
  a.write_from = std::min(T - 1, (int)h->window_size + 1);  // rounds after which cluster_cpp may stop (:250-256)
  a.has_next_from = T - 1;
  a.ring_rows = u.ring_rows;
  a.coop = 1;
  if (t0 == 0 && !rem_ready) {
    // removal sums of round 0 from the R in memory (assignment step / user), harmony.cpp:312-313
    RegionScope r0(h, "k_rem_sums");
    k_rem_sums<<<dim3(h->coop_grid, nb), 256, sizeof(float) * 8 * (size_t)h->KS, h->stream>>>(
        h->R.p, a.order, a.ranges, a.tuple_levels, a.acc, 0, h->coop_grid, h->K, h->KS, h->C, h->B);
    CKL();
    if (h->world > 1) TRY(allreduce_f(h, u.slot(1), u.slot_floats() * nb));  // rem halves of slots 1 .. nb (add halves: zero)
  }
  if (h->world <= 1 || u.use_xch) {
    a.s_begin = t0 * nb;
    a.s_end = t1 * nb;
    RegionScope r3(h, "k_update_steps");
    TRY(launch_single_pass(h, a, true));
  } else {
    // sharded cells without peer memory: one launch per block step, the step's add half all-reduced in between; the next round's
    // removal sums (remT) are all-reduced and folded once per round
    RegionScope r3(h, "k_update_steps");
    for (int t = t0; t < t1; ++t) {
      if (t > 0) {
        TRY(allreduce_f(h, u.remT.p + (size_t)(t & 1) * nb * h->J * h->KS, (size_t)nb * h->J * h->KS));
        k_fold_round<<<grid_for((int64_t)nb * h->K, 256, h->num_sms), 256, 0, h->stream>>>(a, t);
        CKL();
      }
      for (int s = t * nb; s < (t + 1) * nb; ++s) {
        if (s > t0 * nb) TRY(allreduce_f(h, u.slot(s + 1), u.XH));  // add_{s-1}
        a.s_begin = s;
        a.s_end = s + 1;
        TRY(launch_single_pass(h, a, false));
      }
    }
    TRY(allreduce_f(h, u.slot(t1 * nb + 1), u.XH));  // add_{S-1}
  }
  {
    RegionScope r4(h, "k_update_finalize");
    k_single_pass_finalize<<<grid_for(u.BK, 256, 64), 256, 0, h->stream>>>(a, u.use_xch ? u.xch : PeerXch{}, t1 * nb, h->O.p, h->E.p);
    CKL();
  }
  return push_round_objectives(h, t0, t1);
}
// two-pass kernel (update_two_pass.cuh): look-ahead + update warp groups.  rounds [t0, t1): t0 == 0 runs the
// prologue look-ahead.  write_mask: rounds that store R.
int run_update_two_pass(hb_handle* h, int T, int t0, int t1, unsigned write_mask) {
  RegionScope rs(h, "update_R");
  const UpdateState& u = *h->upd;
  const int nb = h->nb;
  const PlanRound0 r = plan_round0(h, h->plan->set);
  TwoPassArgs a = persistent_args<TwoPassArgs>(h, T, r);
  a.seg_start = r.seg_start;
  a.prev_at = r.prev_at;
  a.Psave = u.Psave.p;
  a.first_round_from_R = h->R_user_set ? 1 : 0;
  a.write_R_mask = write_mask;
  if (h->world <= 1) {
    a.s_begin = t0 * nb;
    a.s_end = t1 * nb;
    a.prologue = (t0 == 0) ? 1 : 0;
    RegionScope r3(h, "k_update_steps");
    TRY(launch_two_pass(h, a, true));
  } else {
    // sharded cells: one launch per step, the step's slot [add_{s-1} | rem_s] all-reduced in between
    RegionScope r3(h, "k_update_steps");
    if (t0 == 0) {
      a.s_begin = a.s_end = 0;
      a.prologue = 1;
      TRY(launch_two_pass(h, a, false));
    }
    a.prologue = 0;
    for (int s = t0 * nb; s < t1 * nb; ++s) {
      TRY(allreduce_f(h, u.slot(s + 1), u.slot_floats()));
      a.s_begin = s;
      a.s_end = s + 1;
      TRY(launch_two_pass(h, a, false));
    }
    TRY(allreduce_f(h, u.slot(t1 * nb + 1), u.slot_floats()));  // slot(S): add_{S-1} (+ look-ahead rem_S)
  }
  // tables at the end of round t1-1 -> O, E (the chain itself continues from the ring)
  {
    RegionScope r4(h, "k_update_finalize");
    k_two_pass_finalize<<<grid_for(u.BK, 256, 64), 256, 0, h->stream>>>(a, t1 * nb, h->O.p, h->E.p);
    CKL();
  }
  return push_round_objectives(h, t0, t1);
}

}  // namespace
