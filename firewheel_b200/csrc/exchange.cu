// exchange.cu — hand-over between the processor's main stream and the side stream that carries the master-bus exchange
// between ranks (SURVEY §8e).
//
// The exchange of call e (ncclAllGather of the per-rank buses + the top levels of the tree, runtime.cu: run_bus_stage) runs
// on a high-priority side stream so that it overlaps control + chain of call e + 1. What it needs from the main stream is
// "the rank-local bus of call e is complete". A CUDA event recorded on the main stream would say that, but an event between
// two kernels cuts their programmatic-dependent-launch overlap. Instead:
//   signal    the last CTA of the combine kernel that completes the rank-local bus publishes e in a device word (kernels.cu:
//             combine_kernel, done_word); K-signal below does the same as a one-warp PDL kernel when there is no combine level
//             (<= 64 voices: the chain kernel writes the bus itself);
//   K-wait    (side stream): one warp polls that word until it reaches e; the all-gather is enqueued behind it.
// The main stream therefore carries no event at all in steady state; a poll that exceeds ~2 s raises the plan's error word
// instead of hanging the GPU.
//
// The payload is 512 KiB per rank, far below where store bandwidth matters: NCCL's single low-latency all-gather kernel is
// used rather than a hand-written peer-memory exchange (push + system fence + wait + receive).
#include <cuda_runtime.h>

#include <cstdint>

#include "device.cuh"
#include "kernels.cuh"
#include "plan.hpp"

namespace fw {
namespace {

__global__ void __launch_bounds__(32) bus_signal_kernel(uint32_t* word, uint32_t epoch) {
    pdl_launch_dependents();  // the next call's control kernel follows like any kernel of the chain
    pdl_wait();               // the rank-local bus is complete
    if (threadIdx.x == 0) { __threadfence(); st_release_gpu(word, epoch); }
}

// wait until *word >= epoch (wrapping compare)
__global__ void __launch_bounds__(32) bus_wait_kernel(const uint32_t* word, uint32_t epoch, uint32_t* error, uint32_t error_value) {
    if (threadIdx.x != 0) return;
    const long long t0 = clock64();
    while ((int32_t)(ld_acquire_gpu(word) - epoch) < 0) {
        __nanosleep(200);
        if (clock64() - t0 > 4000000000ll) { *error = error_value; return; }  // ~2 s at 2 GHz
    }
}

}  // namespace

cudaError_t launch_bus_signal(uint32_t* word, uint32_t epoch, cudaStream_t st) {
    return launch_ex(bus_signal_kernel, dim3(1), dim3(32), 0, st, true, word, epoch);
}
cudaError_t launch_bus_wait(const uint32_t* word, uint32_t epoch, uint32_t* error, uint32_t error_value, cudaStream_t st) {
    bus_wait_kernel<<<1, 32, 0, st>>>(word, epoch, error, error_value);
    return cudaGetLastError();
}

}  // namespace fw
