// trace.cuh — the objective trace (appended on the device, mirrored on the host lazily) and the convergence test.
#pragma once

namespace {

int ensure_trace_cap(hb_handle* h, int slots) {
  if (slots <= h->trace_cap) return 0;
  int ncap = std::max(1024, h->trace_cap * 2);
  while (ncap < slots) ncap *= 2;
  float* np = nullptr;
  CK(cudaMalloc((void**)&np, sizeof(float) * 4 * (size_t)ncap));
  if (h->trace_d.p && h->obj_count > 0)
    CK(cudaMemcpyAsync(np, h->trace_d.p, sizeof(float) * 4 * (size_t)h->obj_count, cudaMemcpyDeviceToDevice, h->stream));
  CK(cudaStreamSynchronize(h->stream));
  if (h->trace_d.p) cudaFree(h->trace_d.p);
  h->trace_d.p = np;
  h->trace_d.n = 4 * (size_t)ncap;
  h->trace_cap = ncap;
  return 0;
}

// obj holds this rank's per-cell sums; fold in the K x B cross term of tables (O, E) and append to the trace
int push_objective_from(hb_handle* h, const float* O, const float* E, double* obj) {
  TRY(ensure_trace_cap(h, h->obj_count + 1));
  TRY(allreduce_d(h, obj, 2));
  k_objective_finalize<<<1, 256, 0, h->stream>>>(O, E, h->theta.p, h->sigma.p, obj, h->trace_d.p, h->obj_count, h->B,
                                                  h->K, h->KS, (double)h->N_global, 1.0);
  CKL();
  h->obj_count++;
  return 0;
}
int push_objective(hb_handle* h) { return push_objective_from(h, h->O.p, h->E.p, h->obj_acc.p); }

int sync_traces(hb_handle* h) {
  if (h->obj_synced == h->obj_count) return 0;
  h->obj_vals.resize(4 * (size_t)h->obj_count);
  CK(cudaMemcpyAsync(h->obj_vals.data() + 4 * (size_t)h->obj_synced, h->trace_d.p + 4 * (size_t)h->obj_synced,
                     sizeof(float) * 4 * (size_t)(h->obj_count - h->obj_synced), cudaMemcpyDeviceToHost, h->stream));
  CK(cudaStreamSynchronize(h->stream));
  h->obj_synced = h->obj_count;
  return 0;
}

// harmony.cpp:173-205
int check_convergence_host(hb_handle* h, int type, int* out) {
  TRY(sync_traces(h));
  float obj_new = 0, obj_old = 0;
  auto ok = [&](int slot) { return h->obj_vals[4 * (size_t)slot]; };
  switch (type) {
    case 0: {
      if (h->obj_count < (int)h->window_size + 1) return fail(h, 3, "check_convergence(0): not enough objective values");
      for (unsigned i = 0; i < h->window_size; i++) {
        obj_old += ok(h->obj_count - 2 - (int)i);
        obj_new += ok(h->obj_count - 1 - (int)i);
      }
      *out = (std::abs(obj_old - obj_new) / std::abs(obj_old) < h->epsilon_kmeans) ? 1 : 0;
      return 0;
    }
    case 1: {
      if (h->harmony_slots.size() < 2) return fail(h, 3, "check_convergence(1): not enough objective values");
      obj_old = ok(h->harmony_slots[h->harmony_slots.size() - 2]);
      obj_new = ok(h->harmony_slots[h->harmony_slots.size() - 1]);
      *out = ((obj_old - obj_new) / std::abs(obj_old) < h->epsilon_harmony) ? 1 : 0;
      return 0;
    }
  }
  *out = 1;
  return 0;
}

}  // namespace
