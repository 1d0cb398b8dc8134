// learner_core.cu -- the library-wide error buffer, kernel trace and per-kernel profiler, the packed <-> padded
// parameter copies, and the learner-handle core shared by every learner handle (learner_core.cuh).
#include <stdarg.h>
#include <string.h>

#include <string>

#include "learner_core.cuh"

namespace drl {

static thread_local char g_err[1024] = {0};
void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}
const char* get_error() { return g_err; }

static std::vector<TraceSetter>& trace_setters() {
  static std::vector<TraceSetter> v;
  return v;
}
int register_trace_setter(TraceSetter f) {
  trace_setters().push_back(f);
  return (int)trace_setters().size();
}

// ---- per-kernel profiler -------------------------------------------------------------------
struct Profiler {
  bool on = false;
  std::vector<cudaEvent_t> ev;
  std::vector<const char*> names;
};
static Profiler g_prof;
void prof_mark(cudaStream_t s, const char* name) {
  if (!g_prof.on) return;
  cudaEvent_t e = nullptr;
  if (cudaEventCreate(&e) != cudaSuccess) return;
  cudaEventRecord(e, s);
  g_prof.ev.push_back(e);
  g_prof.names.push_back(name);
}

void prof_begin() {
  g_prof.on = true;
  g_prof.ev.clear();
  g_prof.names.clear();
}
int prof_end(cudaStream_t s, int rc, char* names, int64_t names_len, float* ms, int32_t max_kernels, int32_t* count) {
  g_prof.on = false;
  cudaError_t e = cudaStreamSynchronize(s);
  int n = 0;
  std::string joined;
  if (rc == DRL_OK && e == cudaSuccess) {
    for (size_t i = 0; i + 1 < g_prof.ev.size() && n < max_kernels; ++i) {
      float t = 0.f;
      cudaEventElapsedTime(&t, g_prof.ev[i], g_prof.ev[i + 1]);
      ms[n++] = t;
      if (!joined.empty()) joined += "\n";
      joined += g_prof.names[i];
    }
  }
  for (cudaEvent_t ev : g_prof.ev) cudaEventDestroy(ev);
  g_prof.ev.clear();
  g_prof.names.clear();
  if (rc != DRL_OK) return rc;
  if (e != cudaSuccess) { set_error("profile step failed: %s", cudaGetErrorString(e)); return DRL_ERR_CUDA; }
  if ((int64_t)joined.size() + 1 > names_len) { set_error("profile: names buffer too small"); return DRL_ERR_INVALID; }
  memcpy(names, joined.c_str(), joined.size() + 1);
  *count = n;
  return DRL_OK;
}

int upload_flat(cudaStream_t s, float* h_flat, const FlatLayout& pl, float* dev_padded, const float* host_packed,
                float pad_value) {
  for (int64_t i = 0; i < pl.padded_total; ++i) h_flat[i] = pad_value;
  for (int i = 0; i < pl.num_tensors; ++i)
    memcpy(h_flat + pl.padded_off[i], host_packed + pl.packed_off[i], pl.count[i] * sizeof(float));
  DRL_CUDA_CHECK(cudaMemcpyAsync(dev_padded, h_flat, pl.padded_total * sizeof(float), cudaMemcpyHostToDevice, s));
  DRL_CUDA_CHECK(cudaStreamSynchronize(s));
  return DRL_OK;
}
int download_flat(cudaStream_t s, float* h_flat, const FlatLayout& pl, const float* dev_padded, float* host_packed) {
  DRL_CUDA_CHECK(cudaMemcpyAsync(h_flat, dev_padded, pl.padded_total * sizeof(float), cudaMemcpyDeviceToHost, s));
  DRL_CUDA_CHECK(cudaStreamSynchronize(s));
  for (int i = 0; i < pl.num_tensors; ++i)
    memcpy(host_packed + pl.packed_off[i], h_flat + pl.padded_off[i], pl.count[i] * sizeof(float));
  return DRL_OK;
}

// ---- handle core ----------------------------------------------------------------------------

Streams LearnerCore::streams() const {
  Streams st;
  st.main = compute;
  st.side = side;
  for (int i = 0; i < 8; ++i) st.ev[i] = fj[i];
  st.par = par;
  return st;
}

int learner_core_init(LearnerCore* h, size_t slot_bytes) {
  DRL_CUDA_CHECK(cudaSetDevice(h->device));
  DRL_CUDA_CHECK(cudaStreamCreateWithFlags(&h->compute, cudaStreamNonBlocking));
  DRL_CUDA_CHECK(cudaStreamCreateWithFlags(&h->copy, cudaStreamNonBlocking));
  DRL_CUDA_CHECK(cudaStreamCreateWithFlags(&h->side, cudaStreamNonBlocking));
  for (int i = 0; i < 8; ++i) DRL_CUDA_CHECK(cudaEventCreateWithFlags(&h->fj[i], cudaEventDisableTiming));
  DRL_CUDA_CHECK(cudaEventCreate(&h->ev_start));
  DRL_CUDA_CHECK(cudaEventCreate(&h->ev_stop));
  const size_t NP = h->layout->padded_total;
  DRL_TRY(dev_alloc(h, &h->params, NP));
  DRL_TRY(dev_alloc(h, &h->grads, NP + 4));
  h->loss = h->grads + NP;
  DRL_TRY(dev_alloc(h, &h->d_step, 1));
  DRL_TRY(dev_alloc(h, &h->d_lr, 1));
  const size_t rows = (size_t)h->num_slots + 1;
  DRL_CUDA_CHECK(cudaHostAlloc((void**)&h->h_out, rows * 8 * sizeof(float), cudaHostAllocMapped));
  DRL_CUDA_CHECK(cudaHostGetDevicePointer((void**)&h->d_out, h->h_out, 0));
  memset(h->h_out, 0, rows * 8 * sizeof(float));
  h->ev_done.resize(rows, nullptr);
  for (auto& e : h->ev_done) DRL_CUDA_CHECK(cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
  DRL_CUDA_CHECK(cudaHostAlloc((void**)&h->h_flat, NP * sizeof(float), cudaHostAllocDefault));
  h->slots.resize(h->num_slots + h->scratch_slots);
  h->graph_step.assign(h->num_slots, nullptr);
  h->graph_fb.assign(h->num_slots, nullptr);
  for (LearnerSlot& s : h->slots) {
    DRL_TRY(dev_alloc(h, &s.base, slot_bytes));
    DRL_CUDA_CHECK(cudaEventCreateWithFlags(&s.staged, cudaEventDisableTiming));
    DRL_CUDA_CHECK(cudaEventCreateWithFlags(&s.consumed, cudaEventDisableTiming));
  }
  return DRL_OK;
}

void learner_core_release(LearnerCore* h) {
  cudaSetDevice(h->device);
  cudaDeviceSynchronize();
  for (auto g : h->graph_step) if (g) cudaGraphExecDestroy(g);
  for (auto g : h->graph_fb) if (g) cudaGraphExecDestroy(g);
  if (h->graph_apply) cudaGraphExecDestroy(h->graph_apply);
  for (LearnerSlot& s : h->slots) {
    if (s.staged) cudaEventDestroy(s.staged);
    if (s.consumed) cudaEventDestroy(s.consumed);
  }
  for (void* p : h->allocs) cudaFree(p);
  if (h->h_out) cudaFreeHost(h->h_out);
  if (h->h_flat) cudaFreeHost(h->h_flat);
  for (auto e : h->ev_done) if (e) cudaEventDestroy(e);
  if (h->ev_start) cudaEventDestroy(h->ev_start);
  if (h->ev_stop) cudaEventDestroy(h->ev_stop);
  for (int i = 0; i < 8; ++i) if (h->fj[i]) cudaEventDestroy(h->fj[i]);
  if (h->side) cudaStreamDestroy(h->side);
  if (h->compute) cudaStreamDestroy(h->compute);
  if (h->copy) cudaStreamDestroy(h->copy);
  cudaGetLastError();
}

int set_device(const LearnerCore* h) {
  DRL_CUDA_CHECK(cudaSetDevice(h->device));
  return DRL_OK;
}

int check_handle(const LearnerCore* h, const char* family) {
  if (!h) { set_error("null %s handle", family); return DRL_ERR_INVALID; }
  return DRL_OK;
}

int check_slot(const LearnerCore* h, int slot) {
  if (slot < 0 || slot >= h->num_slots) { set_error("slot %d out of range", slot); return DRL_ERR_INVALID; }
  return DRL_OK;
}

int learner_upload(LearnerCore* h, float* dev_padded, const float* host_packed, float pad_value) {
  DRL_CUDA_CHECK(cudaStreamSynchronize(h->compute));
  return upload_flat(h->compute, h->h_flat, *h->layout, dev_padded, host_packed, pad_value);
}
int learner_download(LearnerCore* h, const float* dev_padded, float* host_packed) {
  return download_flat(h->compute, h->h_flat, *h->layout, dev_padded, host_packed);
}

namespace {

int wait_staged(LearnerCore* h, int slot) {
  const LearnerSlot& sl = h->slots[slot];
  if (!sl.has_data) { set_error("slot %d has not been staged", slot); return DRL_ERR_STATE; }
  DRL_CUDA_CHECK(cudaStreamWaitEvent(h->compute, sl.staged, 0));
  return DRL_OK;
}

int enqueue_fwd_bwd(LearnerCore* h, int slot, int* launches) {
  h->images_stale = true;   // the forward rebuilds the weight images: the last update changed the parameters
  return h->fwd_bwd(h, slot, launches);
}

int enqueue_update(LearnerCore* h, int out_row, float grad_scale, bool local_only, bool early, int* launches) {
  DRL_TRY(h->update(h, out_row, grad_scale, local_only, early));
  if (launches) *launches += 2;
  return DRL_OK;
}

// an update was enqueued into result row `row`: record the events wait / last_step_ms read
int finish_update(LearnerCore* h, int row) {
  h->images_stale = true;
  h->last_row = row;
  DRL_CUDA_CHECK(cudaEventRecord(h->ev_stop, h->compute));
  DRL_CUDA_CHECK(cudaEventRecord(h->ev_done[row], h->compute));
  h->pending = true;
  return DRL_OK;
}

int collect(LearnerCore* h, int row, const float** out) {
  DRL_CUDA_CHECK(cudaEventSynchronize(h->ev_done[row]));
  *out = h->h_out + 8 * row;
  return DRL_OK;
}

}  // namespace

// Under use_cuda_graph, forward + backward and the update go into ONE graph per slot (nothing on the host runs between
// them); the scalars land in the slot's own result row.
int learner_run_step(LearnerCore* h, int slot) {
  DRL_TRY(wait_staged(h, slot));
  DRL_CUDA_CHECK(cudaEventRecord(h->ev_start, h->compute));
  int cnt = 0;
  auto pass = [&] {
    DRL_TRY(enqueue_fwd_bwd(h, slot, &cnt));
    return enqueue_update(h, slot, 1.0f, false, true, &cnt);
  };
  if (h->use_cuda_graph) {
    if (!h->graph_step[slot]) {
      // eager pass of forward + loss + backward first (sets the per-kernel attributes outside of capture; it does not
      // change any state the captured pass depends on: parameters and optimizer state are only touched by the update)
      DRL_TRY(enqueue_fwd_bwd(h, slot, nullptr));
      DRL_TRY(capture_graph(h->compute, pass, &h->graph_step[slot]));
      h->launches = cnt;
    }
    NvtxRange r("drl:step(graph)");
    DRL_CUDA_CHECK(cudaGraphLaunch(h->graph_step[slot], h->compute));
  } else {
    DRL_TRY(pass());
    h->launches = cnt;
  }
  h->last_n = h->B;
  h->last_slot = slot;
  DRL_CUDA_CHECK(cudaEventRecord(h->slots[slot].consumed, h->compute));
  return finish_update(h, slot);
}

int64_t step_of(const float* row) {
  uint32_t lo, hi;
  memcpy(&lo, &row[6], 4);
  memcpy(&hi, &row[7], 4);
  return (int64_t)(((uint64_t)hi << 32) | lo);
}

int learner_param_count(const LearnerCore* h, const char* family, int64_t* n) {
  DRL_TRY(check_handle(h, family));
  std::lock_guard<std::recursive_mutex> lk(h->mu);
  if (!n) { set_error("null argument"); return DRL_ERR_INVALID; }
  *n = h->layout->packed_total;
  return DRL_OK;
}

int learner_set_params(LearnerCore* h, const char* family, const float* host_flat, int64_t n) {
  DRL_TRY(check_handle(h, family));
  std::lock_guard<std::recursive_mutex> lk(h->mu);
  const int64_t np = h->layout->packed_total;
  if (!host_flat || n != np) { set_error("set_params: expected %lld floats, got %lld", (long long)np, (long long)n); return DRL_ERR_INVALID; }
  DRL_TRY(set_device(h));
  DRL_TRY(learner_upload(h, h->params, host_flat, 0.0f));
  h->images_stale = true;
  return DRL_OK;
}

int learner_get_params(LearnerCore* h, const char* family, float* host_flat, int64_t n) {
  DRL_TRY(check_handle(h, family));
  std::lock_guard<std::recursive_mutex> lk(h->mu);
  const int64_t np = h->layout->packed_total;
  if (!host_flat || n != np) { set_error("get_params: expected %lld floats", (long long)np); return DRL_ERR_INVALID; }
  DRL_TRY(set_device(h));
  return learner_download(h, h->params, host_flat);
}

int learner_get_grads(LearnerCore* h, const char* family, const float* bucket, float* host_flat, int64_t n) {
  DRL_TRY(check_handle(h, family));
  std::lock_guard<std::recursive_mutex> lk(h->mu);
  const int64_t np = h->layout->packed_total;
  if (!host_flat || n != np) { set_error("get_grads: expected %lld floats", (long long)np); return DRL_ERR_INVALID; }
  DRL_TRY(set_device(h));
  return learner_download(h, bucket, host_flat);
}

int learner_grad_bucket(LearnerCore* h, const char* family, void** dev_ptr, int64_t* count) {
  DRL_TRY(check_handle(h, family));
  std::lock_guard<std::recursive_mutex> lk(h->mu);
  if (dev_ptr) *dev_ptr = h->grads;
  if (count) *count = h->layout->padded_total + 4;
  return DRL_OK;
}

int learner_params_snapshot(LearnerCore* h, const char* family, int device, cudaStream_t dst_stream, float* dst,
                            cudaEvent_t ev_ready, cudaEvent_t ev_copied) {
  DRL_TRY(check_handle(h, family));
  std::lock_guard<std::recursive_mutex> lk(h->mu);
  if (h->device != device) {
    set_error("sync: the learner is on device %d, the policy on device %d (no cross-device sync)", h->device, device);
    return DRL_ERR_INVALID;
  }
  DRL_TRY(set_device(h));
  NvtxRange r("drl:learner_snapshot");
  DRL_CUDA_CHECK(cudaEventRecord(ev_ready, h->compute));
  DRL_CUDA_CHECK(cudaStreamWaitEvent(dst_stream, ev_ready, 0));
  DRL_CUDA_CHECK(cudaMemcpyAsync(dst, h->params, (size_t)h->layout->padded_total * sizeof(float),
                                 cudaMemcpyDeviceToDevice, dst_stream));
  DRL_CUDA_CHECK(cudaEventRecord(ev_copied, dst_stream));
  DRL_CUDA_CHECK(cudaStreamWaitEvent(h->compute, ev_copied, 0));
  return DRL_OK;
}

int learner_step_async(LearnerCore* h, const char* family, int slot) {
  DRL_TRY(check_handle(h, family));
  std::lock_guard<std::recursive_mutex> lk(h->mu);
  DRL_TRY(check_slot(h, slot));
  DRL_TRY(set_device(h));
  return learner_run_step(h, slot);
}

int learner_forward_backward(LearnerCore* h, const char* family, int slot) {
  DRL_TRY(check_handle(h, family));
  std::lock_guard<std::recursive_mutex> lk(h->mu);
  DRL_TRY(check_slot(h, slot));
  DRL_TRY(set_device(h));
  DRL_TRY(wait_staged(h, slot));
  DRL_CUDA_CHECK(cudaEventRecord(h->ev_start, h->compute));
  int cnt = 0;
  if (h->use_cuda_graph) {
    if (!h->graph_fb[slot]) {
      DRL_TRY(enqueue_fwd_bwd(h, slot, nullptr));   // eager pass: per-kernel attributes are set outside of capture
      DRL_TRY(capture_graph(h->compute, [&] { return enqueue_fwd_bwd(h, slot, &cnt); }, &h->graph_fb[slot]));
      h->launches = cnt + 2;
    }
    DRL_CUDA_CHECK(cudaGraphLaunch(h->graph_fb[slot], h->compute));
  } else {
    DRL_TRY(enqueue_fwd_bwd(h, slot, &cnt));
    h->launches = cnt + 2;
  }
  h->last_n = h->B;
  h->last_slot = slot;
  DRL_CUDA_CHECK(cudaEventRecord(h->slots[slot].consumed, h->compute));
  return DRL_OK;
}

int learner_apply(LearnerCore* h, const char* family, float grad_scale) {
  DRL_TRY(check_handle(h, family));
  std::lock_guard<std::recursive_mutex> lk(h->mu);
  if (!(grad_scale > 0.f)) { set_error("apply: grad_scale must be > 0"); return DRL_ERR_INVALID; }
  DRL_TRY(set_device(h));
  const int row = h->num_slots;
  if (h->use_cuda_graph) {
    if (h->graph_apply && h->graph_apply_scale != grad_scale) {   // the scale is a kernel argument inside the graph
      cudaGraphExecDestroy(h->graph_apply);
      h->graph_apply = nullptr;
    }
    if (!h->graph_apply) {
      DRL_TRY(capture_graph(h->compute, [&] { return enqueue_update(h, row, grad_scale, false, false, nullptr); },
                            &h->graph_apply));
      h->graph_apply_scale = grad_scale;
    }
    DRL_CUDA_CHECK(cudaGraphLaunch(h->graph_apply, h->compute));
  } else {
    DRL_TRY(enqueue_update(h, row, grad_scale, false, false, nullptr));
  }
  return finish_update(h, row);
}

int learner_wait(LearnerCore* h, const char* family, const float** row) {
  DRL_TRY(check_handle(h, family));
  std::lock_guard<std::recursive_mutex> lk(h->mu);
  if (!h->pending) { set_error("wait: no step in flight"); return DRL_ERR_STATE; }
  DRL_TRY(set_device(h));
  h->pending = false;
  return collect(h, h->last_row, row);
}

int learner_wait_slot(LearnerCore* h, const char* family, int slot, const float** row) {
  DRL_TRY(check_handle(h, family));
  std::lock_guard<std::recursive_mutex> lk(h->mu);
  DRL_TRY(check_slot(h, slot));
  DRL_TRY(set_device(h));
  if (slot == h->last_row) h->pending = false;
  return collect(h, slot, row);
}

int learner_profile_step(LearnerCore* h, const char* family, int slot, char* names, int64_t names_len, float* ms,
                         int32_t max_kernels, int32_t* count) {
  DRL_TRY(check_handle(h, family));
  std::lock_guard<std::recursive_mutex> lk(h->mu);
  DRL_TRY(check_slot(h, slot));
  if (!names || !ms || !count) { set_error("null argument"); return DRL_ERR_INVALID; }
  DRL_TRY(set_device(h));
  DRL_TRY(wait_staged(h, slot));
  DRL_CUDA_CHECK(cudaStreamSynchronize(h->compute));
  prof_begin();
  const bool par_saved = h->par;
  h->par = false;                       // serial: the event-to-event times are then per kernel
  int rc = enqueue_fwd_bwd(h, slot, nullptr);
  if (rc == DRL_OK) rc = enqueue_update(h, h->num_slots, 1.0f, /*local_only=*/true, false, nullptr);   // one rank may profile alone
  h->par = par_saved;
  h->images_stale = true;
  h->last_n = h->B;
  DRL_TRY(prof_end(h->compute, rc, names, names_len, ms, max_kernels, count));
  h->pending = false;
  return DRL_OK;
}

int learner_last_step_ms(LearnerCore* h, const char* family, float* ms) {
  DRL_TRY(check_handle(h, family));
  std::lock_guard<std::recursive_mutex> lk(h->mu);
  if (!ms) { set_error("null argument"); return DRL_ERR_INVALID; }
  DRL_TRY(set_device(h));
  DRL_CUDA_CHECK(cudaEventSynchronize(h->ev_stop));
  DRL_CUDA_CHECK(cudaEventElapsedTime(ms, h->ev_start, h->ev_stop));
  return DRL_OK;
}

int learner_stream(LearnerCore* h, const char* family, void** stream) {
  DRL_TRY(check_handle(h, family));
  std::lock_guard<std::recursive_mutex> lk(h->mu);
  if (!stream) { set_error("null argument"); return DRL_ERR_INVALID; }
  *stream = h->compute;
  return DRL_OK;
}

int learner_launches_per_step(const LearnerCore* h, const char* family, int32_t* n) {
  DRL_TRY(check_handle(h, family));
  std::lock_guard<std::recursive_mutex> lk(h->mu);
  if (!n) { set_error("null argument"); return DRL_ERR_INVALID; }
  *n = h->launches;     // valid after the first step
  return DRL_OK;
}

int read_named_buffer(LearnerCore* h, const NamedBuffer* tab, int ntab, const char* name, float* host_dst, int64_t n) {
  for (int i = 0; i < ntab; ++i) {
    const NamedBuffer& e = tab[i];
    if (strcmp(e.name, name) != 0) continue;
    if ((size_t)n != e.count) { set_error("read_buffer(%s): expected %zu floats, got %lld", name, e.count, (long long)n); return DRL_ERR_INVALID; }
    if (e.p == nullptr) { set_error("read_buffer(%s): not kept in this math mode", name); return DRL_ERR_INVALID; }
    DRL_CUDA_CHECK(cudaStreamSynchronize(h->compute));
    DRL_CUDA_CHECK(cudaMemcpy(host_dst, e.p, e.count * sizeof(float), cudaMemcpyDeviceToHost));
    return DRL_OK;
  }
  set_error("read_buffer: unknown buffer '%s'", name);
  return DRL_ERR_INVALID;
}

}  // namespace drl

extern "C" {

const char* drl_last_error(void) { return drl::get_error(); }

// debug: arm (dev_buf = device buffer of >= 8001 uint64, word 0 = entry counter) or disarm (NULL) the kernel
// start-time trace of common.cuh::kernel_prologue
int drl_debug_trace(void* dev_buf) {
  if (drl_device_count() < 1) { drl::set_error("CUDA device not available (no CPU fallback)"); return DRL_ERR_CUDA; }
  DRL_CUDA_CHECK(cudaDeviceSynchronize());
  for (drl::TraceSetter f : drl::trace_setters()) f(static_cast<unsigned long long*>(dev_buf));
  DRL_CUDA_CHECK(cudaDeviceSynchronize());
  return DRL_OK;
}
const char* drl_version(void) { return "drl_b200 0.5 (sm_90a; wgmma split-16 / 3xTF32 gather-GEMMs, FP32-FFMA core, NVLink peer exchange; IMPALA, Ape-X, R2D2, A3C learners)"; }

int drl_device_count(void) {
  int n = 0;
  if (cudaGetDeviceCount(&n) != cudaSuccess) { cudaGetLastError(); return 0; }
  return n;
}

}  // extern "C"
