// kernels.cuh — launchers for kernels.cu (all asynchronous on the given stream).
#pragma once
#include <cuda_runtime.h>

#include <cstddef>
#include <cstdint>

#include <string>

#include "plan.hpp"

namespace fw {
cudaError_t launch_control(ControlArgs a, cudaStream_t st);
uint32_t control_threads(uint32_t n_flag_words, int device);  // CTA size of the control kernel, 0: the flags of one voice do not fit
cudaError_t launch_chain(const ChainArgs& a, bool bus, cudaStream_t st);
uint32_t chain_voice_groups(uint32_t num_voices);  // partial buses produced by the bus variant
cudaError_t launch_sum(const SumArgs& a, cudaStream_t st);
cudaError_t launch_resampler(const ResamplerArgs& a, uint64_t* pos, cudaStream_t st);  // data kernel + position advance
cudaError_t launch_sampler(const SamplerArgs& a, cudaStream_t st);
cudaError_t launch_silence_fix(const SilenceFixArgs& a, cudaStream_t st);
cudaError_t launch_expand_masks(const Records& rec, uint32_t mask_slot, uint32_t V, uint32_t n_blocks, uint64_t* out, cudaStream_t st);
cudaError_t launch_combine(const float* pin, float* pout, uint32_t n_in, uint32_t rows, uint32_t T, cudaStream_t st, uint32_t out_pitch = 0,
                           uint32_t* done_word = nullptr, uint32_t* done_counter = nullptr, uint32_t done_epoch = 0);  // done_*: see combine_kernel
cudaError_t launch_deinterleave(const float* inter, float* planar, uint32_t V, uint32_t C, uint32_t T, cudaStream_t st);
cudaError_t launch_interleave(const float* planar, float* inter, const uint64_t* masks, uint32_t V, uint32_t C, uint32_t T,
                              uint32_t block_frames, cudaStream_t st);
cudaError_t launch_fill(float* p, size_t n, float val, cudaStream_t st);
// +0.0 into `rows` rows of T frames (pitch row_pitch floats) in each of `groups` groups (pitch group_pitch floats) from p
cudaError_t launch_zero_rows(float* p, uint32_t T, uint64_t row_pitch, uint32_t rows, uint32_t groups, uint64_t group_pitch, cudaStream_t st);
cudaError_t launch_bus_mask(const uint64_t* gout_mask, uint32_t V, uint32_t n_out, uint64_t* bus_mask, cudaStream_t st);
cudaError_t launch_bus_signal(uint32_t* word, uint32_t epoch, cudaStream_t st);
cudaError_t launch_bus_wait(const uint32_t* word, uint32_t epoch, uint32_t* error, uint32_t error_value, cudaStream_t st);
cudaError_t launch_poke(const PokeArgs& a, cudaStream_t st);
cudaError_t launch_temporal(const TemporalArgs& a, cudaStream_t st);
uint32_t reverb_kpad(uint32_t L);
uint32_t reverb_hist(uint32_t L);
uint32_t reverb_grid_max();   // CTAs of the persistent GEMM grid (= SMs)
size_t reverb_ws_bytes();      // tail-wave fix-up workspace per ConvReverb node
cudaError_t launch_reverb_build(const float* d_ir, void* d_bt, uint32_t L, uint32_t ir_ch, cudaStream_t st);
cudaError_t launch_reverb(const ReverbCall& rc, cudaStream_t st, std::string* err);
}  // namespace fw
