// b2_context.cu -- library state, error reporting, context (device + stream + staging).
#include <atomic>
#include <cstring>

#include "b2_internal.hpp"

namespace b2 {

static thread_local char g_last_error[1024] = "";

b2_status fail(b2_status st, const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_last_error, sizeof(g_last_error), fmt, ap);
  va_end(ap);
  return st;
}

namespace {
// cuCtxGetCurrent and cuCtxSetCurrent, looked up once through the runtime: the library does not link libcuda, so it still loads on
// a machine without a driver, where b2_ctx_create reports B2_ERR_NO_DEVICE before any scope is opened.  NULL if the lookup failed.
struct CtxCalls {
  CUresult (*get)(CUcontext*) = nullptr;
  CUresult (*set)(CUcontext) = nullptr;
};
const CtxCalls* ctx_calls() {
  static const CtxCalls calls = [] {
    CtxCalls c;
    void* fn = nullptr;
    cudaDriverEntryPointQueryResult found;
    if (cudaGetDriverEntryPoint("cuCtxGetCurrent", &fn, cudaEnableDefault, &found) == cudaSuccess && found == cudaDriverEntryPointSuccess)
      c.get = reinterpret_cast<CUresult (*)(CUcontext*)>(fn);
    if (cudaGetDriverEntryPoint("cuCtxSetCurrent", &fn, cudaEnableDefault, &found) == cudaSuccess && found == cudaDriverEntryPointSuccess)
      c.set = reinterpret_cast<CUresult (*)(CUcontext)>(fn);
    return c;
  }();
  return calls.get && calls.set ? &calls : nullptr;
}
}  // namespace

DeviceScope::DeviceScope(int device) {
  const CtxCalls* calls = ctx_calls();
  if (!calls) {
    status_ = fail(B2_ERR_CUDA, "cudaGetDriverEntryPoint: cuCtxGetCurrent / cuCtxSetCurrent not found");
    return;
  }
  const CUresult r = calls->get(&saved_);
  if (r != CUDA_SUCCESS) {
    status_ = fail(B2_ERR_CUDA, "cuCtxGetCurrent -> CUresult %d", static_cast<int>(r));
    return;
  }
  restore_ = true;
  const cudaError_t e = cudaSetDevice(device);
  if (e != cudaSuccess) {
    status_ = fail(e == cudaErrorMemoryAllocation ? B2_ERR_OUT_OF_MEMORY : B2_ERR_CUDA, "cudaSetDevice(%d) -> %s", device, cudaGetErrorString(e));
    return;
  }
  CUcontext now = nullptr;
  restore_ = calls->get(&now) != CUDA_SUCCESS || now != saved_;  // the common case: the device was current already
}

DeviceScope::~DeviceScope() {
  if (restore_) ctx_calls()->set(saved_);
}

// ---- residency ----

namespace {
std::atomic<uint64_t> g_access_clock{0};
}  // namespace

uint64_t access_clock_now() { return g_access_clock.load(); }
uint64_t access_clock_tick() { return g_access_clock.fetch_add(1); }

b2_status offload_arrays(std::initializer_list<DeviceBuffer*> bufs, std::initializer_list<size_t> sizes, cudaStream_t st, HostCopy& host) {
  size_t total = 0;
  for (size_t s : sizes) total += s;
  HostCopy h;
  B2_TRY(h.block.alloc(total));
  size_t off = 0;
  auto s = sizes.begin();
  for (DeviceBuffer* b : bufs) {
    const size_t bytes = *b ? *s : 0;
    if (bytes) B2_CUDA(cudaMemcpyAsync(h.block.get() + off, b->get(), bytes, cudaMemcpyDeviceToHost, st));
    h.sizes.push_back(bytes);
    h.alloc.push_back(b->bytes());
    off += bytes;
    ++s;
  }
  B2_CUDA(cudaStreamSynchronize(st));
  host.block = std::move(h.block);
  host.sizes = std::move(h.sizes);
  host.alloc = std::move(h.alloc);
  return B2_OK;
}

b2_status reload_arrays(std::initializer_list<DeviceBuffer*> bufs, std::initializer_list<bool> zero, cudaStream_t st, const HostCopy& host) {
  // everything is allocated and queued before any buffer is handed over: on failure `fresh` frees what was allocated here
  std::vector<DeviceBuffer> fresh(bufs.size());
  size_t off = 0;
  auto z = zero.begin();
  for (size_t k = 0; k < fresh.size(); k++, ++z) {
    if (host.alloc[k] > 0) {
      B2_TRY(fresh[k].alloc(host.alloc[k]));
      if (*z) B2_CUDA(cudaMemsetAsync(fresh[k].get(), 0, host.alloc[k], st));
      if (host.sizes[k]) B2_CUDA(cudaMemcpyAsync(fresh[k].get(), host.block.get() + off, host.sizes[k], cudaMemcpyHostToDevice, st));
    }
    off += host.sizes[k];
  }
  size_t k = 0;
  for (DeviceBuffer* b : bufs) *b = std::move(fresh[k++]);
  return B2_OK;
}

b2_status stream_after(cudaStream_t other, cudaStream_t st) {
  if (other == st) return B2_OK;
  cudaEvent_t ev = nullptr;
  B2_CUDA(cudaEventCreateWithFlags(&ev, cudaEventDisableTiming));
  cudaError_t e = cudaEventRecord(ev, st);
  if (e == cudaSuccess) e = cudaStreamWaitEvent(other, ev, 0);
  cudaEventDestroy(ev);  // released once the wait has been satisfied
  B2_CUDA(e);
  return B2_OK;
}

}  // namespace b2

b2_status b2_ctx::ensure_stage(size_t host_bytes) {
  // the new buffer is allocated BEFORE the old one is released: a failed allocation leaves the context usable
  if (host_bytes > h_stage_bytes) {
    const size_t want = b2::round_up(host_bytes * 2, 4096);
    void* fresh = nullptr;
    B2_CUDA(cudaHostAlloc(&fresh, want, cudaHostAllocMapped | cudaHostAllocPortable));
    if (h_stage) {
      cudaStreamSynchronize(stream);  // nothing in flight may still read the old staging area
      cudaFreeHost(h_stage);
    }
    h_stage = fresh;
    h_stage_bytes = want;
  }
  return B2_OK;
}

extern "C" {

const char* b2_last_error(void) { return b2::g_last_error; }
const char* b2_version(void) { return "b2points 0.1 (sm_90a)"; }

b2_status b2_ctx_create(int device, void* stream, b2_ctx** out) {
  B2_REQUIRE(out != nullptr, "b2_ctx_create: out is NULL");
  *out = nullptr;
  int count = 0;
  cudaError_t e = cudaGetDeviceCount(&count);
  if (e != cudaSuccess || count == 0) {
    // No CPU fallback exists anywhere in this library: without a CUDA device nothing can run.
    return b2::fail(B2_ERR_NO_DEVICE, "b2_ctx_create: no CUDA device available (%s)", e != cudaSuccess ? cudaGetErrorString(e) : "count = 0");
  }
  B2_REQUIRE(device >= 0 && device < count, "b2_ctx_create: device %d out of range [0, %d)", device, count);
  const b2::DeviceScope on_device(device);
  B2_TRY(on_device.status());
  b2_ctx* ctx = new b2_ctx;
  ctx->device = device;
  if (stream) {
    ctx->stream = static_cast<cudaStream_t>(stream);
    ctx->owns_stream = false;
  } else {
    cudaError_t es = cudaStreamCreateWithFlags(&ctx->stream, cudaStreamNonBlocking);
    if (es != cudaSuccess) {
      delete ctx;
      return b2::fail(B2_ERR_CUDA, "cudaStreamCreateWithFlags: %s", cudaGetErrorString(es));
    }
    ctx->owns_stream = true;
  }
  cudaDeviceProp prop;
  cudaError_t ep = cudaGetDeviceProperties(&prop, device);
  if (ep != cudaSuccess) {
    delete ctx;
    return b2::fail(B2_ERR_CUDA, "cudaGetDeviceProperties: %s", cudaGetErrorString(ep));
  }
  ctx->sm_count = prop.multiProcessorCount;
  {
    // completion word for zero-copy host calls: pinned + mapped, plus the device counter that decides who writes it
    void* h = nullptr;
    void* d = nullptr;
    cudaError_t ed = cudaHostAlloc(&h, 64, cudaHostAllocMapped | cudaHostAllocPortable);
    if (ed == cudaSuccess) ed = cudaHostGetDevicePointer(&d, h, 0);
    if (ed == cudaSuccess) ed = cudaMalloc(reinterpret_cast<void**>(&ctx->d_done_counter), sizeof(unsigned int));
    if (ed == cudaSuccess) ed = cudaMemset(ctx->d_done_counter, 0, sizeof(unsigned int));
    if (ed != cudaSuccess) {
      if (h) cudaFreeHost(h);
      if (ctx->d_done_counter) cudaFree(ctx->d_done_counter);
      if (ctx->owns_stream) cudaStreamDestroy(ctx->stream);
      delete ctx;
      return b2::fail(B2_ERR_CUDA, "b2_ctx_create: completion word: %s", cudaGetErrorString(ed));
    }
    *static_cast<volatile unsigned int*>(h) = 0u;
    ctx->h_done = static_cast<volatile unsigned int*>(h);
    ctx->d_done_flag = static_cast<volatile unsigned int*>(d);
  }
  *out = ctx;
  return B2_OK;
}

b2_status b2_ctx_destroy(b2_ctx* ctx) {
  if (!ctx) return B2_OK;
  const b2::DeviceScope on_device(ctx->device);
  cudaStreamSynchronize(ctx->stream);
  if (ctx->h_stage) cudaFreeHost(ctx->h_stage);
  if (ctx->h_done) cudaFreeHost(const_cast<unsigned int*>(ctx->h_done));
  if (ctx->d_done_counter) cudaFree(ctx->d_done_counter);
  if (ctx->owns_stream) cudaStreamDestroy(ctx->stream);
  delete ctx;
  return B2_OK;
}

b2_status b2_ctx_synchronize(b2_ctx* ctx) {
  B2_REQUIRE(ctx != nullptr, "b2_ctx_synchronize: ctx is NULL");
  B2_ON_DEVICE(ctx);  // a runtime call on a thread without a current context would make device 0's primary context current
  B2_CUDA(cudaStreamSynchronize(ctx->stream));
  return B2_OK;
}

void* b2_ctx_stream(b2_ctx* ctx) { return ctx ? static_cast<void*>(ctx->stream) : nullptr; }

b2_status b2_access_time_current(uint64_t* out) {
  B2_REQUIRE(out != nullptr, "b2_access_time_current: out is NULL");
  *out = b2::access_clock_now();
  return B2_OK;
}

b2_status b2_device_malloc(b2_ctx* ctx, size_t bytes, void** out) {
  B2_REQUIRE(ctx && out, "b2_device_malloc: NULL argument");
  *out = nullptr;
  B2_ON_DEVICE(ctx);
  B2_CUDA(cudaMalloc(out, bytes ? bytes : 1));
  return B2_OK;
}

b2_status b2_device_free(b2_ctx* ctx, void* ptr) {
  B2_REQUIRE(ctx != nullptr, "b2_device_free: ctx is NULL");
  if (!ptr) return B2_OK;
  B2_ON_DEVICE(ctx);
  B2_CUDA(cudaStreamSynchronize(ctx->stream));
  B2_CUDA(cudaFree(ptr));
  return B2_OK;
}

b2_status b2_memcpy_d2h(b2_ctx* ctx, void* dst, const void* src, size_t bytes) {
  B2_REQUIRE(ctx && (bytes == 0 || (dst && src)), "b2_memcpy_d2h: NULL argument");
  B2_ON_DEVICE(ctx);
  B2_CUDA(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToHost, ctx->stream));
  B2_CUDA(cudaStreamSynchronize(ctx->stream));
  return B2_OK;
}

b2_status b2_memcpy_h2d(b2_ctx* ctx, void* dst, const void* src, size_t bytes) {
  B2_REQUIRE(ctx && (bytes == 0 || (dst && src)), "b2_memcpy_h2d: NULL argument");
  B2_ON_DEVICE(ctx);
  B2_CUDA(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyHostToDevice, ctx->stream));
  B2_CUDA(cudaStreamSynchronize(ctx->stream));
  return B2_OK;
}

}  // extern "C"
