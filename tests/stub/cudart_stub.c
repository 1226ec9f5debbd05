/* tests/stub/cudart_stub.c — TEST TOOLING ONLY, never linked into the product.
 * A stand-in for the handful of CUDA runtime calls libcrgpu's HOST code makes (device memory = malloc, copies = memcpy,
 * kernel launches = no-ops), so that the host half of crgpu_scene_create — validation, BVH re-layout into pair nodes,
 * triangle packing, shading records — can be exercised, timed and its upload bytes pinned in the CPU test suite
 * (tests/test_create_host.py), and so that the edit calls' block bookkeeping can be checked (tests/test_edit_blocks_host.py).
 * Nothing is rendered: there is no CPU path for the kernels. */
#include <stdlib.h>
#include <string.h>
#include <stdio.h>
#include <time.h>
#include <stdint.h>
static double now_(void){struct timespec t;clock_gettime(CLOCK_MONOTONIC,&t);return t.tv_sec+1e-9*t.tv_nsec;}
static double t_last; static uint64_t g_sum=1469598103934665603ull; static int g_trace=-1;
static void note(const char*what,const void*src,size_t n){ if(g_trace<0) g_trace=getenv("STUB_TRACE")?1:0; double t=now_(); if(src && !getenv("STUB_NOHASH")){const unsigned char*p=src; uint64_t h=1469598103934665603ull; /* per upload */ for(size_t i=0;i<n;i+=1){h=(h^p[i])*1099511628211ull;} g_sum=h;} if(g_trace) fprintf(stderr,"%8.2f ms since prev  %-10s %zu bytes  sum %016llx\n",1e3*(t-t_last),what,n,(unsigned long long)g_sum); t_last=now_(); }
unsigned long long stub_checksum(void){return g_sum;}
void stub_reset(void){g_sum=1469598103934665603ull; t_last=now_();}
typedef int cudaError_t; typedef void *cudaStream_t; typedef void *cudaEvent_t;
struct cudaDeviceProp_stub { char pad[4096]; };
cudaError_t cudaGetDeviceCount(int *n) { *n = 1; return 0; }
cudaError_t cudaSetDevice(int d) { (void)d; return 0; }
cudaError_t cudaGetDevice(int *d) { *d = 0; return 0; }
cudaError_t cudaDeviceSynchronize(void) { note("devsync",0,0); return 0; }
cudaError_t cudaGetLastError(void) { return 0; }
const char *cudaGetErrorString(cudaError_t e) { (void)e; return "stub"; }
/* device allocations still live, and a switch that fails cudaMalloc from its k-th call on (tests/stub/edit_blocks_harness.c) */
static long g_live, g_mallocs, g_fail_from = -1;
long stub_live_allocs(void) { return g_live; }
void stub_fail_malloc_from(long k) { g_mallocs = 0; g_fail_from = k; }   /* k counts calls from now, 1-based; k < 0 lifts it */
cudaError_t cudaMalloc(void **p, size_t n) {
	if (g_fail_from >= 0 && ++g_mallocs >= g_fail_from) { *p = NULL; return 2; }   /* cudaErrorMemoryAllocation */
	*p = malloc(n ? n : 1);
	if (*p) ++g_live;
	return *p ? 0 : 2;
}
cudaError_t cudaFree(void *p) { if (p) --g_live; free(p); return 0; }
cudaError_t cudaHostAlloc(void **p, size_t n, unsigned f) { (void)f; *p = malloc(n ? n : 1); return *p ? 0 : 2; }
cudaError_t cudaFreeHost(void *p) { free(p); return 0; }
cudaError_t cudaMemcpy(void *d, const void *s, size_t n, int k) { (void)k; note("memcpy",s,n); memcpy(d, s, n); t_last=now_(); return 0; }
cudaError_t cudaMemcpyAsync(void *d, const void *s, size_t n, int k, cudaStream_t st) { (void)k; (void)st; memcpy(d, s, n); return 0; }
cudaError_t cudaMemcpy2DAsync(void *d, size_t dp, const void *s, size_t sp, size_t w, size_t h, int k, cudaStream_t st) { (void)k; (void)st; for (size_t y = 0; y < h; ++y) memcpy((char *)d + y * dp, (const char *)s + y * sp, w); return 0; }
cudaError_t cudaMemset(void *d, int v, size_t n) { memset(d, v, n); return 0; }
cudaError_t cudaMemsetAsync(void *d, int v, size_t n, cudaStream_t st) { (void)st; memset(d, v, n); return 0; }
cudaError_t cudaMemGetInfo(size_t *f, size_t *t) { *f = (size_t)170 << 30; *t = (size_t)180 << 30; return 0; }
cudaError_t cudaStreamCreateWithFlags(cudaStream_t *s, unsigned f) { (void)f; *s = (void *)1; return 0; }
cudaError_t cudaStreamDestroy(cudaStream_t s) { (void)s; return 0; }
cudaError_t cudaStreamSynchronize(cudaStream_t s) { (void)s; return 0; }
cudaError_t cudaEventCreate(cudaEvent_t *e) { *e = (void *)1; return 0; }
cudaError_t cudaEventCreateWithFlags(cudaEvent_t *e, unsigned f) { (void)f; *e = (void *)1; return 0; }
cudaError_t cudaStreamWaitEvent(cudaStream_t s, cudaEvent_t e, unsigned f) { (void)s; (void)e; (void)f; return 0; }
cudaError_t cudaEventDestroy(cudaEvent_t e) { (void)e; return 0; }
cudaError_t cudaEventRecord(cudaEvent_t e, cudaStream_t s) { (void)e; (void)s; return 0; }
cudaError_t cudaEventElapsedTime(float *ms, cudaEvent_t a, cudaEvent_t b) { (void)a; (void)b; *ms = 0; return 0; }
cudaError_t cudaDeviceGetAttribute(int *v, int a, int d) { (void)a; (void)d; *v = 148; return 0; }
cudaError_t cudaFuncSetAttribute(const void *f, int a, int v) { (void)f; (void)a; (void)v; return 0; }
cudaError_t cudaOccupancyMaxActiveBlocksPerMultiprocessorWithFlags(int *n, const void *f, int b, size_t s, unsigned fl) { (void)f; (void)b; (void)s; (void)fl; *n = 3; return 0; }
cudaError_t cudaGetDeviceProperties_v2(void *prop, int d) { (void)d; memset(prop, 0, 1032); /* multiProcessorCount filled by the caller of this stub via env */ 
	int *p = (int *)prop; const char *off = getenv("STUB_SM_OFFSET"); if (off) p[atoi(off) / 4] = 148; return 0; }
cudaError_t cudaLaunchKernel(const void *f, ...) { (void)f; return 0; }
unsigned __cudaPushCallConfiguration(void) { return 0; }
cudaError_t __cudaPopCallConfiguration(void *a, void *b, size_t *c, void *d) { (void)a; (void)b; (void)c; (void)d; return 0; }
void **__cudaRegisterFatBinary(void *p) { (void)p; static void *h; return &h; }
void __cudaRegisterFatBinaryEnd(void **h) { (void)h; }
void __cudaUnregisterFatBinary(void **h) { (void)h; }
void __cudaRegisterFunction(void **h, const char *a, char *b, const char *c, int d, void *e, void *f, void *g, void *i, int *j) { (void)h; (void)a; (void)b; (void)c; (void)d; (void)e; (void)f; (void)g; (void)i; (void)j; }
