// Grid-wide barrier for kernels whose CTAs are all co-resident (one per SM, cooperative launch): the recurrent steps of the
// tensor-core LSTM kernels (encodec.cu).
//
// One monotonic 32-bit counter: after its CTA-level barrier ONE thread per CTA arrives with a gpu-scope release
// reduction (no return value: the L2 atomic unit does not answer) and polls with gpu-scope acquire loads until the count
// reaches phase * gridDim.  The CTA barrier in front makes the release cumulative over every thread's earlier global
// writes (PTX memory model, release pattern through bar.sync); the CTA barrier behind hands the acquire to the rest of
// the CTA.  The caller zeroes the counter in front of the kernel, so targets never wrap inside a launch.
#pragma once
#include <stdint.h>

__device__ __forceinline__ void gridbar_arrive(unsigned* ctr) {
    asm volatile("red.release.gpu.global.add.u32 [%0], 1;" ::"l"(ctr) : "memory");
}
__device__ __forceinline__ unsigned gridbar_load_acquire(const unsigned* ctr) {
    unsigned v;
    asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(ctr) : "memory");
    return v;
}
__device__ __forceinline__ void gridbar_wait(const unsigned* ctr, unsigned target) {
    while (gridbar_load_acquire(ctr) < target) { }
}
