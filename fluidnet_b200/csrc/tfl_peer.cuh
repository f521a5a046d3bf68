// The signalling protocol of every exchange between processes over CUDA IPC mappings (the z-slab halos and
// all-reduce, the z-slab frame recorder, the step monitor's mapped host records).
//
// A writer stores its data with plain stores, fences at system scope (__threadfence_system), then stores a sequence
// number into a word with release semantics at system scope.  A reader loads that word with acquire semantics at
// system scope until it has reached the number it waits for; what the writer stored before the word is then visible.
// Sequence numbers only grow and are compared wrap-safe: a word has reached `target` once (int)(v - target) >= 0.
// Waits are bounded by kPeerWaitCycles: a peer that never arrives makes the wait return false instead of hanging the
// GPU, and the caller decides what a timeout does (raise the fault counter, skip the data, mark the rank missing).
#pragma once

constexpr int kMaxRanks = 64;                       // ranks sharing peer memory: one thread each in a one-block wait,
                                                    // one bit each in the recorder's 64-bit missing-rank mask
constexpr long long kPeerWaitCycles = 4000000000LL; // a wait's bound: ~2 s at the H100's clock

__device__ __forceinline__ void store_release_sys(unsigned int* word, unsigned int v) {
  asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(word), "r"(v) : "memory");
}
__device__ __forceinline__ void store_release_sys(unsigned long long* word, unsigned long long v) {
  asm volatile("st.release.sys.global.u64 [%0], %1;" ::"l"(word), "l"(v) : "memory");
}

// This thread's earlier stores, then `seq` in `word`.
__device__ __forceinline__ void publish_seq(unsigned int* word, unsigned int seq) {
  __threadfence_system();
  store_release_sys(word, seq);
}

// Polls `word` (sleeping sleep_ns between loads) until it reaches `target`: true, and the writer's stores before it are
// visible; false once kPeerWaitCycles have passed since clock64() read t0.
__device__ __forceinline__ bool wait_seq(const unsigned int* word, unsigned int target, long long t0, unsigned int sleep_ns) {
  for (;;) {
    unsigned int v;
    asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(word) : "memory");
    if ((int)(v - target) >= 0) return true;
    if (clock64() - t0 > kPeerWaitCycles) return false;
    __nanosleep(sleep_ns);
  }
}

// Called by every thread of every CTA of a grid of `blocks` CTAs after its stores: once every CTA's stores are fenced,
// the last CTA to count itself in `done` (zero between launches) resets it and publishes `seq` in word0 and word1
// (null: skipped).  `leader` is one thread per CTA.
__device__ __forceinline__ void last_cta_publish(unsigned int* done, unsigned int blocks, bool leader, unsigned int* word0,
                                                 unsigned int* word1, unsigned int seq) {
  __threadfence_system();
  __syncthreads();
  if (leader && atomicAdd(done, 1u) == blocks - 1) {
    *done = 0u;
    __threadfence_system();
    if (word0) store_release_sys(word0, seq);
    if (word1) store_release_sys(word1, seq);
  }
}
