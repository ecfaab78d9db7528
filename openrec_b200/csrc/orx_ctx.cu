// orx_ctx.cu -- context, workspace and error plumbing of liborx.
#include <stdarg.h>
#include <stdlib.h>
#include <string.h>

#include "orx_common.cuh"

static thread_local char g_err[512] = "";

void orx_set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}

extern "C" const char* orx_last_error_string(void) { return g_err; }

bool orx_pdl_enabled() {
  static int v = -1;
  if (v < 0) {
    const char* e = getenv("ORX_PDL");
    v = (e && atoi(e) == 0) ? 0 : 1;
  }
  return v != 0;
}
extern "C" int orx_abi_version(void) { return ORX_ABI_VERSION; }

extern "C" int orx_device_count(int* n) {
  ORX_REQUIRE(n != nullptr, "null output");
  *n = 0;
  ORX_CUDA(cudaGetDeviceCount(n));
  return ORX_OK;
}

uint32_t orx_hash_shape(OrxHash& t, int64_t lookups) {
  // load factor <= 0.25: with linear probing the slowest of a warp's 32 inserts/probes sets the pace
  // (profile r1b: ~7 serialized L2 round trips per warp at 0.5)
  uint32_t cap = 1024;
  while ((int64_t)cap < 4 * lookups) cap <<= 1;
  int lg = 0;
  while ((1u << lg) < cap) ++lg;
  t.mask = cap - 1;
  t.shift = 32 - lg;
  return cap;
}

void orx_hash_carve(OrxCarve& m, OrxHash& t, int64_t lookups) {
  const uint32_t cap = orx_hash_shape(t, lookups);
  t.slots = (unsigned long long*)m.take(sizeof(unsigned long long) * cap);
  t.didx = (int32_t*)m.take(sizeof(int32_t) * cap);
  t.did = (int32_t*)m.take(sizeof(int32_t) * (size_t)(lookups + 1));
}

// The index workspace for nb lookups on the user side and 2 nb on the item side: the control words of the three index
// sets side by side, their tables and the records of sets 1 and 2, then the staging rows gu | gi | gb | gw.  Every
// lookup may be staged (ADAM_DENSE stages all rows), so the staging rows hold nb resp. 2 nb rows of nd floats.  With
// base == nullptr only the size is computed, and every pointer is left null.
static size_t index_ws_layout(char* base, int64_t nb, int32_t nd, orx_ctx* c) {
  OrxCarve m = {base, 0};
  int32_t* ctl = (int32_t*)m.take(sizeof(int32_t) * 4 * 3);
  for (int k = 0; k < 3; ++k) {
    OrxIndexSet& s = c->set[k];
    s.ctl = base ? ctl + 4 * k : nullptr;
    s.u.counter = s.ctl;
    s.i.counter = base ? s.ctl + 1 : nullptr;
    orx_hash_carve(m, s.u, nb);
    orx_hash_carve(m, s.i, 2 * nb);
    s.res = k > 0 && c->pair_resolve ? (int4*)m.take(sizeof(int4) * (size_t)nb) : nullptr;
  }
  c->gu = (float*)m.take(sizeof(float) * (size_t)nb * nd);
  c->gi = (float*)m.take(sizeof(float) * 2 * (size_t)nb * nd);
  c->gb = (float*)m.take(sizeof(float) * 2 * (size_t)nb);
  c->gw = (float*)m.take(sizeof(float) * (size_t)nd);
  return m.off;
}

int orx_ensure_workspace(orx_ctx* c, int64_t B, int32_t dim) {
  if (B <= c->cap_B && dim <= c->g_dim) return ORX_OK;
  const int64_t nb = B > c->cap_B ? B : c->cap_B;
  const int32_t nd = dim > c->g_dim ? dim : c->g_dim;
  ORX_CUDA(cudaDeviceSynchronize());   // the old layout may be in use on any stream
  // until the new layout is in place: no set points into the old buffer, and a failed allocation is retried next call
  c->cap_B = 0;
  c->g_dim = 0;
  const size_t bytes = index_ws_layout(nullptr, nb, nd, c);
  int rc = orx_grow(&c->index_ws, &c->index_cap, bytes);
  if (rc) return rc;
  index_ws_layout(static_cast<char*>(c->index_ws), nb, nd, c);
  ORX_CUDA(cudaMemset(c->index_ws, 0, bytes));
  // the memset ran on the legacy default stream; the caller's stream may be a non-blocking one
  ORX_CUDA(cudaDeviceSynchronize());
  for (OrxIndexSet& s : c->set) {
    s.u.epoch = s.i.epoch = 0;  // fresh (zeroed) tables: epochs restart at 1
    s.free_valid = 0;
  }
  c->pf_set = 0;
  c->cap_B = nb;
  c->g_dim = nd;
  return ORX_OK;
}

int orx_take_epoch(OrxHash& t, cudaStream_t st) {
  const uint32_t e = (t.epoch + 1) & 0x7fffffffu;
  if (e == 0) ORX_CUDA(cudaMemsetAsync(t.slots, 0, sizeof(unsigned long long) * ((size_t)t.mask + 1), st));
  t.epoch = e ? e : 1;
  return ORX_OK;
}

// test hook: place the epoch of every index table, the handle's, orx_censor_shard's and the sharded step's (the wrap
// tests start them just below 2^31)
extern "C" int orx_debug_set_epoch(orx_handle_t h, uint32_t epoch) {
  ORX_REQUIRE(h != nullptr && epoch < 0x80000000u, "null handle / epoch must be < 2^31");
  for (OrxIndexSet& s : h->set) s.u.epoch = s.i.epoch = epoch;
  h->censor_hash.epoch = epoch;
  orx_shard_set_epoch(h, epoch);
  return ORX_OK;
}

// test hook: which kernel each DLRM entry point and sparse step launched (tests/test_gpu_dlrm.py and
// tests/test_gpu_kernels.py assert the dispatch of every case)
extern "C" int orx_debug_dispatch_log(orx_handle_t h, int32_t* rec, int32_t cap, int32_t* n) {
  ORX_REQUIRE(h != nullptr && n && cap >= 0 && (rec || cap == 0), "bad arguments");
  const int64_t held = h->dispatch_n < ORX_DISPATCH_LOG_CAP ? h->dispatch_n : ORX_DISPATCH_LOG_CAP;
  const int64_t first = h->dispatch_n - held;   // oldest record still in the ring
  const int64_t take = held < cap ? held : cap;
  for (int64_t i = 0; i < take; ++i) memcpy(rec + 8 * i, h->dispatch[(first + i) % ORX_DISPATCH_LOG_CAP], 8 * sizeof(int32_t));
  *n = (int32_t)take;
  h->dispatch_n = 0;
  return ORX_OK;
}

int orx_grow(void** buf, size_t* cap, size_t need) {
  if (need <= *cap) return ORX_OK;
  ORX_CUDA(cudaDeviceSynchronize());
  cudaFree(*buf);
  *buf = nullptr;
  *cap = 0;
  const cudaError_t e = cudaMalloc(buf, need);
  if (e != cudaSuccess) {
    cudaGetLastError();   // not left behind for the next launch check to report
    *buf = nullptr;
    orx_set_error("workspace allocation of %zu bytes failed: %s", need, cudaGetErrorString(e));
    return ORX_ERR_NOMEM;
  }
  *cap = need;
  return ORX_OK;
}

extern "C" int orx_create(int device, orx_handle_t* out) {
  ORX_REQUIRE(out != nullptr, "null output handle");
  *out = nullptr;
  int n = 0;
  ORX_CUDA(cudaGetDeviceCount(&n));
  ORX_REQUIRE(device >= 0 && device < n, "device ordinal out of range");
  ORX_CUDA(cudaSetDevice(device));
  cudaDeviceProp prop;
  ORX_CUDA(cudaGetDeviceProperties(&prop, device));
  if (prop.major != 9 || prop.minor != 0) {
    orx_set_error("orx_create: liborx is built for sm_90a only; device %d is sm_%d%d", device, prop.major,
                  prop.minor);
    return ORX_ERR_UNSUPPORTED;
  }
  orx_ctx* c = new orx_ctx();
  memset(c, 0, sizeof(*c));
  c->device = device;
  c->num_sms = prop.multiProcessorCount;
  c->partials_cap = sizeof(float) * 2 * (size_t)c->num_sms * 64;
  const char* pr = getenv("ORX_PAIR_RESOLVE");   // 0: prefetched pairwise steps probe the index (A/B measurements)
  c->pair_resolve = (pr && atoi(pr) == 0) ? 0 : 1;
  if (cudaMalloc(&c->bucket_cursor, sizeof(int32_t) * 1024) != cudaSuccess ||
      cudaMalloc(&c->partials, c->partials_cap) != cudaSuccess ||
      cudaMalloc(&c->out_stage[0], sizeof(float) * 8) != cudaSuccess ||
      cudaMalloc(&c->out_stage[1], sizeof(float) * 8) != cudaSuccess) {
    orx_set_error("orx_create: workspace allocation failed: %s", cudaGetErrorString(cudaGetLastError()));
    orx_destroy(c);
    return ORX_ERR_NOMEM;
  }
  *out = c;
  return ORX_OK;
}

extern "C" int orx_destroy(orx_handle_t h) {
  if (!h) return ORX_OK;
  cudaSetDevice(h->device);
  cudaDeviceSynchronize();
  cudaFree(h->index_ws);
  for (int i = 0; i < 2; ++i) {
    cudaFree(h->ids_stage[i]);
    cudaFree(h->out_stage[i]);
  }
  cudaFree(h->partials);
  cudaFree(h->bucket_cursor);
  cudaFree(h->eval_ws);
  cudaFree(h->lookup_ws);
  cudaFree(h->splitk);
  cudaFree(h->censor_ws);
  cudaFree(h->bag_ws);
  cudaFree(h->bag_cnt_ws);
  cudaFree(h->shard_scratch);
  orx_shard_ws_release(h);
  if (h->side_stream) {
    cudaStreamDestroy(h->side_stream);
    cudaEventDestroy(h->side_ev);
    for (int i = 0; i < 2; ++i) {
      cudaEventDestroy(h->set[1 + i].done);
      cudaEventDestroy(h->set[1 + i].free);
      cudaEventDestroy(h->stage_free[i]);
    }
  }
  if (h->prof_ev) {
    for (int i = 0; i < h->prof_cap * ORX_PROF_EV; ++i) cudaEventDestroy(h->prof_ev[i]);
    delete[] h->prof_ev;
  }
  delete h;
  return ORX_OK;
}

extern "C" int orx_profile_enable(orx_handle_t h, int32_t on) {
  ORX_REQUIRE(h != nullptr, "null handle");
  ORX_CUDA(cudaSetDevice(h->device));
  if (on && !h->prof_ev) {
    h->prof_cap = 1024;
    h->prof_ev = new cudaEvent_t[h->prof_cap * ORX_PROF_EV];
    for (int i = 0; i < h->prof_cap * ORX_PROF_EV; ++i) ORX_CUDA(cudaEventCreate(&h->prof_ev[i]));
  }
  h->prof_on = on ? 1 : 0;
  h->prof_n = 0;
  h->prof_step = 0;
  return ORX_OK;
}

extern "C" int orx_profile_read(orx_handle_t h, float* ms, int32_t n_phases, int32_t* n_steps) {
  ORX_REQUIRE(h != nullptr && ms && n_steps && n_phases >= 1 && n_phases < ORX_PROF_EV, "bad arguments");
  ORX_CUDA(cudaSetDevice(h->device));
  for (int k = 0; k < n_phases; ++k) ms[k] = 0.f;
  *n_steps = h->prof_n;
  for (int i = 0; i < h->prof_n; ++i) {
    ORX_CUDA(cudaEventSynchronize(h->prof_ev[i * ORX_PROF_EV + n_phases]));
    for (int k = 0; k < n_phases; ++k) {
      float t = 0.f;
      ORX_CUDA(cudaEventElapsedTime(&t, h->prof_ev[i * ORX_PROF_EV + k], h->prof_ev[i * ORX_PROF_EV + k + 1]));
      ms[k] += t;
    }
  }
  h->prof_n = 0;
  return ORX_OK;
}

extern "C" int orx_stream_synchronize(orx_handle_t h, orx_stream_t s) {
  ORX_REQUIRE(h != nullptr, "null handle");
  ORX_CUDA(cudaStreamSynchronize((cudaStream_t)s));
  return ORX_OK;
}

bool orx_opt_slots_ok(int kind, std::initializer_list<const orx_table_t*> tabs) {
  // ROWWISE_ADAGRAD needs s0 (float[rows]: its length is the caller's, as for every slot row) and no s1; MOMENTUM and
  // NESTEROV need s0 (a) and no s1
  const bool s0 = kind != ORX_OPT_SGD, s1 = kind == ORX_OPT_ADAM_LAZY || kind == ORX_OPT_ADAM_DENSE;
  for (const orx_table_t* t : tabs)
    if (t && ((s0 && !t->s0) || (s1 && !t->s1))) return false;
  return true;
}

OrxOptDev orx_opt_to_dev(const orx_opt_t* o) {
  OrxOptDev d;
  d.kind = o->kind;
  d.lr = o->lr;
  d.eps = o->eps;
  d.beta1 = o->beta1;
  d.beta2 = o->beta2;
  // SGD, ADAGRAD, ROWWISE_ADAGRAD, MOMENTUM and NESTEROV take lr as given
  if (o->kind == ORX_OPT_ADAM_LAZY || o->kind == ORX_OPT_ADAM_DENSE) {
    // lr_t = lr*sqrt(1-b2^t)/(1-b1^t), evaluated in double like the oracle's adam_lr_t
    double t = (double)(o->step < 1 ? 1 : o->step);
    d.lr = (float)((double)o->lr * sqrt(1.0 - pow((double)o->beta2, t)) / (1.0 - pow((double)o->beta1, t)));
  }
  return d;
}
