// cuda_fake_runtime.cpp — TEST INFRASTRUCTURE: the few CUDA runtime entry points the library calls, implemented on
// the host for the -DB200_EMULATE build (tests/emu/cuda_emu_full.h): device memory is host memory, streams and events
// are synchronous, there is one "device" with 4 SMs.  Linked INSTEAD of libcudart into
// tests/emu/_build/libgtsam_b200_emu.so; never part of the product.
#include <cuda_runtime.h>

#include <chrono>
#include <cstdlib>
#include <cstring>

extern "C" {
cudaError_t cudaGetDeviceCount(int* n) { *n = 1; return cudaSuccess; }
cudaError_t cudaSetDevice(int) { return cudaSuccess; }
cudaError_t cudaGetDeviceProperties_v2(cudaDeviceProp* p, int) { memset(p, 0, sizeof *p); p->multiProcessorCount = 4; return cudaSuccess; }
cudaError_t cudaStreamCreateWithFlags(cudaStream_t* s, unsigned) { *s = (cudaStream_t)0x1; return cudaSuccess; }
cudaError_t cudaStreamDestroy(cudaStream_t) { return cudaSuccess; }
cudaError_t cudaStreamSynchronize(cudaStream_t) { return cudaSuccess; }
// allocation-failure injection (tests/emu/run_scenarios.py allocfail): the live count of cudaMalloc / cudaMallocHost blocks,
// and a countdown after which one allocation fails
static long g_live = 0, g_fail_in = 0;
long b200_emu_live_allocs(void) { return g_live; }
void b200_emu_fail_alloc_in(long k) { g_fail_in = k; }   // the k-th next allocation fails (k >= 1); 0: none
cudaError_t cudaMalloc(void** p, size_t n) {
  *p = nullptr;
  if (g_fail_in > 0 && --g_fail_in == 0) return cudaErrorMemoryAllocation;
  *p = calloc(n ? n : 1, 1);
  if (!*p) return cudaErrorMemoryAllocation;
  g_live++;
  return cudaSuccess;
}
cudaError_t cudaFree(void* p) { if (p) g_live--; free(p); return cudaSuccess; }
cudaError_t cudaMallocHost(void** p, size_t n) { return cudaMalloc(p, n); }
cudaError_t cudaFreeHost(void* p) { return cudaFree(p); }
cudaError_t cudaMemcpyAsync(void* d, const void* s, size_t n, cudaMemcpyKind, cudaStream_t) { if (n) memmove(d, s, n); return cudaSuccess; }
cudaError_t cudaMemcpy(void* d, const void* s, size_t n, cudaMemcpyKind k) { return cudaMemcpyAsync(d, s, n, k, 0); }
cudaError_t cudaMemsetAsync(void* d, int v, size_t n, cudaStream_t) { if (n) memset(d, v, n); return cudaSuccess; }
cudaError_t cudaMemcpyToSymbol(const void* sym, const void* src, size_t n, size_t off, cudaMemcpyKind) { memcpy((char*)sym + off, src, n); return cudaSuccess; }
cudaError_t cudaFuncSetAttribute(const void*, cudaFuncAttribute, int) { return cudaSuccess; }
cudaError_t cudaGetLastError(void) { return cudaSuccess; }
const char* cudaGetErrorString(cudaError_t) { return "emulated CUDA runtime"; }
cudaError_t cudaPointerGetAttributes(cudaPointerAttributes* a, const void*) { memset(a, 0, sizeof *a); a->type = cudaMemoryTypeHost; return cudaSuccess; }
// events: wall clock
struct FakeEvent { double t; };
static double now_ms() { return std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now().time_since_epoch()).count(); }
cudaError_t cudaEventCreate(cudaEvent_t* e) { *e = (cudaEvent_t) new FakeEvent{0}; return cudaSuccess; }
cudaError_t cudaEventDestroy(cudaEvent_t e) { delete (FakeEvent*)e; return cudaSuccess; }
cudaError_t cudaEventRecord(cudaEvent_t e, cudaStream_t) { ((FakeEvent*)e)->t = now_ms(); return cudaSuccess; }
cudaError_t cudaEventElapsedTime(float* ms, cudaEvent_t a, cudaEvent_t b) { *ms = (float)(((FakeEvent*)b)->t - ((FakeEvent*)a)->t); return cudaSuccess; }
// CUDA graphs are not emulated: the library falls back to eager launches when B200_NO_GRAPH is set (the test sets it);
// these stubs only satisfy the linker
cudaError_t cudaStreamBeginCapture(cudaStream_t, cudaStreamCaptureMode) { return cudaErrorNotSupported; }
cudaError_t cudaStreamEndCapture(cudaStream_t, cudaGraph_t* g) { *g = nullptr; return cudaErrorNotSupported; }
cudaError_t cudaGraphInstantiateWithFlags(cudaGraphExec_t*, cudaGraph_t, unsigned long long) { return cudaErrorNotSupported; }
cudaError_t cudaGraphInstantiate(cudaGraphExec_t*, cudaGraph_t, unsigned long long) { return cudaErrorNotSupported; }
cudaError_t cudaGraphDestroy(cudaGraph_t) { return cudaSuccess; }
cudaError_t cudaGraphExecDestroy(cudaGraphExec_t) { return cudaSuccess; }
cudaError_t cudaGraphLaunch(cudaGraphExec_t, cudaStream_t) { return cudaErrorNotSupported; }
}
