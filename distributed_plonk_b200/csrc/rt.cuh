// Runtime shim: the product build is nvcc + the CUDA runtime.  Defining DP_EMUL (done ONLY by
// tests/emul/build.py) swaps in the CPU kernel-logic emulator so tests can run without a GPU.
#pragma once
#if defined(DP_EMUL)
#include "../../tests/emul/cuda_emul.h"
#define DP_LAUNCH(kernel, grid, block, smem, stream, ...) \
    dp_emul::launch_on(stream, grid, block, smem, [=] { kernel(__VA_ARGS__); })
#define DP_DYN_SMEM(name) unsigned char *name = dp_emul::t_dyn_smem
#else
#if !defined(__CUDACC__)
#error "distributed_plonk_b200 is a CUDA library: compile with nvcc for sm_90a (no CPU build exists)"
#endif
#include <cuda_runtime.h>
#define DP_LAUNCH(kernel, grid, block, smem, stream, ...) kernel<<<grid, block, smem, stream>>>(__VA_ARGS__)
#define DP_DYN_SMEM(name) extern __shared__ __align__(128) unsigned char name[]
#endif
#include "field.cuh"
