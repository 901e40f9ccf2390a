// b2t_platform.cuh -- compile-target glue for the tracker kernels.
//
// Product build: nvcc, sm_90a (see build.py).  The B2T_HOSTSIM branch is used ONLY by
// tests/hostsim (a fiber-based single-block simulator for the GPU-less CI tier); the shipped
// library is never built with it.
#pragma once
#include <stdint.h>

#if defined(B2T_HOSTSIM)
#include "cuda_sim.h"
#define B2T_DYN_SMEM(name) unsigned char* name = sim::g.dyn_smem
#define B2T_LAUNCH(kernel, grid, block, smem, stream, ...) \
    sim::launch(dim3(grid), dim3(block), (size_t)(smem), [&] { kernel(__VA_ARGS__); })
#define B2T_SET_SMEM(kernel, bytes) 0
#define B2T_PREFETCH_L1(ptr) ((void)(ptr))
// single-rounded IEEE fp32 operations: the simulator library is built with -ffp-contract=off, so nothing fuses them
inline float __fadd_rn(float a, float b) { return a + b; }
inline float __fsub_rn(float a, float b) { return a - b; }
inline float __fmul_rn(float a, float b) { return a * b; }
inline float __fdiv_rn(float a, float b) { return a / b; }
#else
#include <cuda_runtime.h>
#define B2T_DYN_SMEM(name) extern __shared__ __align__(1024) unsigned char name[]
#define B2T_LAUNCH(kernel, grid, block, smem, stream, ...) kernel<<<(grid), (block), (smem), (stream)>>>(__VA_ARGS__)
#define B2T_SET_SMEM(kernel, bytes) \
    cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(bytes))
#define B2T_PREFETCH_L1(ptr) asm volatile("prefetch.global.L1 [%0];" ::"l"(ptr))
#endif

#define B2T_DEV __device__ __forceinline__
// Everything is force-inlined: out-of-line device functions for the big phases would move their
// by-reference work structs to local memory under the ABI.
#define B2T_DEVNI __device__ __forceinline__
// shared-memory carves: run on the device over the Arena, and on the host over an ArenaSize to size the launch
#define B2T_HD __host__ __device__ __forceinline__
#define B2T_FULL 0xffffffffu
