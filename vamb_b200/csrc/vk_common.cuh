// Shared helpers for the vamb_b200 kernels (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>

#include "../../include/vamb_b200.h"

typedef unsigned long long u64;

void vk_set_error(const char *fmt, ...);

#define VK_CUDA(call)                                                                      \
    do {                                                                                   \
        cudaError_t _e = (call);                                                           \
        if (_e != cudaSuccess) {                                                           \
            vk_set_error("%s:%d: %s -> %s", __FILE__, __LINE__, #call, cudaGetErrorString(_e)); \
            return 1;                                                                      \
        }                                                                                  \
    } while (0)

#define VK_LAUNCH_CHECK()                                                                  \
    do {                                                                                   \
        cudaError_t _e = cudaGetLastError();                                               \
        if (_e != cudaSuccess) {                                                           \
            vk_set_error("%s:%d: kernel launch -> %s", __FILE__, __LINE__, cudaGetErrorString(_e)); \
            return 1;                                                                      \
        }                                                                                  \
    } while (0)

int vk_num_sms();

// 128-byte CUtensorMap (vk_tma.cu) of an fp32 [rows][ld] array, box 32 x box_rows, 128B swizzle; 0 = ok
int vk_make_tmap_2d(void *out128, const float *base, int ld, int rows, int box_rows);
struct alignas(64) VkTmap {
    unsigned char opaque[128];
};

// ---- streaming (read-once) global loads: bypass L1 allocation ----
__device__ __forceinline__ float4 ldg_stream4(const float *p) {
    float4 v;
    asm volatile("ld.global.nc.L1::no_allocate.v4.f32 {%0, %1, %2, %3}, [%4];"
                 : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w)
                 : "l"(p));
    return v;
}

// ---- "vk arithmetic v1": the 8-lane dot product -------------------------------------
// Chunk c (elements 4c..4c+3) belongs to lane (c & 7) of an 8-lane group; every lane runs
// one fmaf chain over its chunks in increasing c; the eight partial sums are combined by
// an xor butterfly (1, 2, 4).  oracle/csrc/oracle_kernels.c:dot8 is the same order.
__device__ __forceinline__ float group8_sum(float acc, unsigned mask) {
    acc = __fadd_rn(acc, __shfl_xor_sync(mask, acc, 1));
    acc = __fadd_rn(acc, __shfl_xor_sync(mask, acc, 2));
    acc = __fadd_rn(acc, __shfl_xor_sync(mask, acc, 4));
    return acc;
}

__device__ __forceinline__ unsigned group8_mask() {
    return 0xFFu << (threadIdx.x & 24);  // lanes of this thread's 8-lane group within its warp
}

// partial (per-lane) chain for generic D; x = row base (global), q = query (shared)
__device__ __forceinline__ float lane_chain_generic(const float *__restrict__ x, const float *q, int d,
                                                    int lane8, bool vec4) {
    float acc = 0.0f;
    const int nchunk = (d + 3) >> 2;
    for (int c = lane8; c < nchunk; c += 8) {
        const int k0 = c << 2;
        if (vec4) {
            const float4 v = ldg_stream4(x + k0);
            const float4 w = *reinterpret_cast<const float4 *>(q + k0);
            acc = __fmaf_rn(v.x, w.x, acc);
            acc = __fmaf_rn(v.y, w.y, acc);
            acc = __fmaf_rn(v.z, w.z, acc);
            acc = __fmaf_rn(v.w, w.w, acc);
        } else {
            const int k1 = min(k0 + 4, d);
            for (int k = k0; k < k1; ++k) acc = __fmaf_rn(__ldg(x + k), q[k], acc);
        }
    }
    return acc;
}

__device__ __forceinline__ float chain4(const float4 v, const float4 w) {
    float acc = __fmaf_rn(v.x, w.x, 0.0f);
    acc = __fmaf_rn(v.y, w.y, acc);
    acc = __fmaf_rn(v.z, w.z, acc);
    acc = __fmaf_rn(v.w, w.w, acc);
    return acc;
}

// closeness (0.05f - d) is always a multiple of 2^-29 -> exact integer in those units
__device__ __forceinline__ u64 closeness_fx(float radius, float d) {
    const float c = __fsub_rn(radius, d);
    return __float2ull_rz(c * 536870912.0f);
}

// exact density accumulation split into two 64-bit sums (see vk_probe_header)
__device__ __forceinline__ void density_add(u64 &lo, u64 &hi, u64 len, u64 cq) {
    lo += len * (cq & 4095ull);
    hi += len * (cq >> 12);
}

// ---- programmatic dependent launch (PDL): the next kernel of the stream may be scheduled while this one
// is still running; it blocks in pdl_wait() until this grid has completed and its memory is visible.
__device__ __forceinline__ void pdl_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
// every kernel of the VAE step starts with this pair (before any global-memory access)
// ---- optional in-kernel timeline (build with -DVK_TIMELINE; tools/step_timeline.py, tools/probe_timeline.py) ----
#ifdef VK_TIMELINE
static __device__ unsigned long long vk_tl[4096];  // per translation unit; vk_vae.cu reads its own
static __device__ int vk_tl_base;
__device__ __forceinline__ void tl_mark(int slot) {
    if (blockIdx.x == 0 && blockIdx.y == 0 && threadIdx.x == 0) {
        unsigned long long t;
        asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
        vk_tl[(vk_tl_base + slot) & 4095] = t;
        vk_tl[((vk_tl_base + slot) & 4095) ^ 2048] = (unsigned long long)clock64();
    }
}
// stamp from thread 0 of WHICHEVER block calls it (e.g. the last block of a mapped-completion kernel)
__device__ __forceinline__ void tl_mark_any(int slot) {
    if (threadIdx.x == 0) {
        unsigned long long t;
        asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
        vk_tl[(vk_tl_base + slot) & 4095] = t;
        vk_tl[((vk_tl_base + slot) & 4095) ^ 2048] = (unsigned long long)clock64();
    }
}
__device__ __forceinline__ void tl_begin(int kernel_id) {
    if (blockIdx.x == 0 && blockIdx.y == 0 && threadIdx.x == 0) vk_tl_base = kernel_id * 64;
    tl_mark(0);
}
// one record per launch, in launch order: [kind, start of block 0, end of block 0, 0]
static __device__ unsigned long long vk_tk[4096 * 4];
static __device__ unsigned int vk_tk_seq;
__device__ __forceinline__ int tk_begin(int kind) {
    if (blockIdx.x == 0 && blockIdx.y == 0 && blockIdx.z == 0 && threadIdx.x == 0) {
        const int idx = (int)(atomicAdd(&vk_tk_seq, 1u) & 4095u);
        unsigned long long t;
        asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
        vk_tk[idx * 4] = (unsigned long long)kind;
        vk_tk[idx * 4 + 1] = t;
        return idx;
    }
    return -1;
}
__device__ __forceinline__ void tk_end(int idx) {
    if (idx >= 0) {
        unsigned long long t;
        asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
        vk_tk[idx * 4 + 2] = t;
    }
}
#else
#define tl_mark(slot) ((void)0)
#define tl_mark_any(slot) ((void)0)
#define tl_begin(id) ((void)0)
#define tk_begin(kind) (-1)
#define tk_end(idx) ((void)(idx))
#endif

__device__ __forceinline__ void pdl_entry() {
    pdl_launch_dependents();
    pdl_wait();
}

bool vk_pdl_enabled();

template <typename... KArgs, typename... Args>
static inline cudaError_t vk_launch(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t s,
                                    Args... args) {
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = grid;
    cfg.blockDim = block;
    cfg.dynamicSmemBytes = smem;
    cfg.stream = s;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr;
    cfg.numAttrs = vk_pdl_enabled() ? 1 : 0;
    return cudaLaunchKernelEx(&cfg, kernel, KArgs(args)...);
}

// as vk_launch, as thread-block clusters of `cluster` CTAs (grid dimensions are multiples of the cluster's)
template <typename... KArgs, typename... Args>
static inline cudaError_t vk_launch_cluster(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t s,
                                            dim3 cluster, Args... args) {
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = grid;
    cfg.blockDim = block;
    cfg.dynamicSmemBytes = smem;
    cfg.stream = s;
    cudaLaunchAttribute attr[2];
    attr[0].id = cudaLaunchAttributeClusterDimension;
    attr[0].val.clusterDim.x = cluster.x;
    attr[0].val.clusterDim.y = cluster.y;
    attr[0].val.clusterDim.z = cluster.z;
    attr[1].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[1].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr;
    cfg.numAttrs = vk_pdl_enabled() ? 2 : 1;
    return cudaLaunchKernelEx(&cfg, kernel, KArgs(args)...);
}
