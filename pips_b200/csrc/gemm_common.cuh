// Shared pieces of the wgmma kernels (gemm_tc.cu, conv_tc.cu, conv_grad.cu, conv_rows.cu, the score-map kernels).
#pragma once
#include <cuda_bf16.h>

#include "common.cuh"
#include "ptx.cuh"

namespace pips {

constexpr int BK = 64;                       // 64 bf16 = one 128-byte swizzle row
constexpr int MMA_K = 16;

// Dynamic shared memory rounded up to 1024 bytes, the alignment 128-byte-swizzled tiles need (launchers reserve 1024
// bytes for it).
__device__ __forceinline__ uint8_t* aligned_smem() {
    extern __shared__ uint8_t smem_raw[];
    return reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~static_cast<uintptr_t>(1023));
}

// The TMA ring: `stages` slots of `slot_bytes` in shared memory, each guarded by a full barrier (its TMA bytes have
// landed) and an empty barrier (every consumer has released it).  The producer and each consumer walk the slots in
// order, each with its own (stage, phase); phase is the parity of the current pass over the ring.
struct Ring {
    uint8_t* slots;
    uint32_t slot_bytes;
    int stages;                             // at run time for conv_tc, whose stage size depends on its tile width
    uint32_t full0, empty0;                 // full[s] at full0 + 8 s, empty[s] at empty0 + 8 s
    uint32_t stage = 0, phase = 0;

    // `bars`: `bar_slots` (>= stages) full barriers, then as many empty ones
    __device__ __forceinline__ Ring(uint8_t* slots_, uint32_t slot_bytes_, int stages_, uint64_t* bars, int bar_slots)
        : slots(slots_), slot_bytes(slot_bytes_), stages(stages_), full0(smem_u32(bars)), empty0(full0 + 8 * bar_slots) {}

    // by one thread, before the barrier that makes the ring visible to the CTA (cluster)
    __device__ __forceinline__ void init(uint32_t consumer_arrivals) const {
        for (int s = 0; s < stages; ++s) {
            mbar_init(full0 + 8 * s, 1);
            mbar_init(empty0 + 8 * s, consumer_arrivals);
        }
        fence_barrier_init();
    }
    __device__ __forceinline__ uint32_t slot() const { return smem_u32(slots + stage * slot_bytes); }
    // producer: waits until the current slot is empty, announces its bytes, issues `load(slot address, full barrier)`
    // (the TMA loads of the slot) and moves to the next slot.  One function, so that the wait's parity is reused as the
    // next pass's phase (a select on the wrap, not an xor): that is the form the GEMM inference kernels had, and it keeps
    // their code unchanged.
    template <typename Load>
    __device__ __forceinline__ void produce(Load&& load) {
        const uint32_t empty_parity = phase ^ 1;
        mbar_wait(empty0 + 8 * stage, empty_parity);
        const uint32_t full = full0 + 8 * stage;
        mbar_arrive_expect_tx(full, slot_bytes);
        load(slot(), full);
        if (++stage == static_cast<uint32_t>(stages)) { stage = 0; phase = empty_parity; }
    }
    // consumer: waits until the current slot has landed; returns its address.  The consumer releases the slot and
    // advances when its policy says so.
    __device__ __forceinline__ uint32_t wait() const {
        mbar_wait(full0 + 8 * stage, phase);
        return slot();
    }
    __device__ __forceinline__ uint32_t empty(uint32_t s) const { return empty0 + 8 * s; }
    __device__ __forceinline__ void release(uint32_t s) const { mbar_arrive(empty(s)); }
    __device__ __forceinline__ void advance() {
        if (++stage == static_cast<uint32_t>(stages)) { stage = 0; phase ^= 1; }
    }
};

// One bf16x3 step: a.b ~= a_hi.b_hi + a_lo.b_hi + a_hi.b_lo into one fp32 accumulator, `mma(a, b, accumulate)` being
// one MMA of the caller's shape.  The bits depend on the order of the three terms; every kernel issues them here.
template <typename Mma, typename A, typename B>
__device__ __forceinline__ void mma_bf16x3(Mma&& mma, A a_hi, A a_lo, B b_hi, B b_lo, uint32_t accumulate) {
    mma(a_hi, b_hi, accumulate);
    mma(a_lo, b_hi, 1u);
    mma(a_hi, b_lo, 1u);
}

}  // namespace pips
