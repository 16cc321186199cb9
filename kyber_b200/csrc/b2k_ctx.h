// b2k_ctx.h -- private definition of the context shared by the translation units of libb2kyber.so.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <string>

constexpr int B2K_N_EV = 12;

// slots of b2k_ctx::last_plan, the layout b2k_last_msm_plan returns (kyber_b200/capi.py: last_msm_plan decodes it)
enum MsmPlanSlot {
  LP_C = 0, LP_W, LP_NB, LP_M,   // window bits, windows, buckets per window, single-level chunk
  LP_SLICE,                      // slice length the XYZZ slices ran with
  LP_ROUNDS,                     // affine rounds
  LP_BATCH,                      // their batch widths, one slot per possible round (8)
  LP_GLV = LP_BATCH + 8,
  LP_SPLIT,                      // affine rounds as three kernels
  LP_LEVELS, LP_M1, LP_M2,       // bucket reduction: levels and chunk per level (LP_M2 = 0 for one level)
  LP_SLOTS = 20
};

struct b2k_arena {
  char* base = nullptr;
  size_t cap = 0, used = 0;
};

struct b2k_ctx {
  int device = 0;
  int sm_count = 132;   // multiprocessors of the device (cudaDeviceProp), sizes the affine rounds of the MSM
  cudaStream_t stream = nullptr;
  bool own_stream = false;
  b2k_arena arena;
  uint32_t* d_flags = nullptr;
  uint32_t* h_flags = nullptr;   // pinned
  cudaEvent_t ev[B2K_N_EV];
  bool timings_valid = false;
  int force_c = 0;
  int force_m = 0;      // bucket-reduction chunk override (0 = automatic)
  int force_L = 0;      // slice length override (0 = automatic)
  int use_glv = 1;      // BLS12-381 G1 MSM: split scalars with the curve endomorphism (0 = plain 255-bit pipeline, for A/B)
  int use_v1 = 0;       // 1 = one-thread-per-bucket accumulate (kept for A/B measurements)
  cudaStream_t stream2 = nullptr;   // high-priority side stream: bucket reduction of one window group overlaps the next accumulate
  cudaStream_t copy_stream = nullptr;   // H2D of the host-buffer MSM in chunks, next to the front-end kernels (msm_host)
  int h2d_chunks = 0;               // > 1 while msm_host enqueues a chunked call: the front end waits for gev[1 + k] before chunk k
  cudaEvent_t gev[10];              // group hand-over events (msm_groups > 1) / chunk hand-over events of the chunked input copy
  int msm_groups = 1;               // window groups of the overlapped MSM tail; measured SLOWER than the serial pipeline
                                    // (accumulate blocks fill the register file, nothing co-resides): kept as an experiment
  int affine_rounds = -1;           // affine pair-tree rounds before the XYZZ slices: -1 = automatic, 0 = off (A/B), 1..8 forced
  int affine_split = 1;             // 1 = every round as three kernels (forward products / inversions / backward additions), 0 = one fused kernel
  int affine_batch = 0;             // outputs (batched affine additions) per thread of a round, 8..64; 0 = automatic
  int mul_minb = 0;                 // BLS12-381 G1 Point.Mul batches: resident blocks per SM (0 = compiler's choice, 3, 4), tuning aid
  int pt_stage = 0;                 // affine rounds with cp.async-staged operands: backward pass bit 0 = round 0 (gather), bit 1 = later rounds; forward pass bits 2, 3
  bool pt_stage_opted = false;      // cudaFuncSetAttribute(MaxDynamicSharedMemorySize) done for the staged backward kernels on this context's device
  int acc_minb = 4;                 // register cap of the inversion kernel of the affine rounds: 4 = uncapped (99 registers), 5 = 96 registers
                                    // (leaves a block slot per SM for another MSM's product kernel: measured no gain);
                                    // b2k_set_msm_occupancy, A/B aid
  int reduce_levels = 0;            // bucket reduction: 0 = automatic (two levels for >= 4096 buckets per window), 1, 2
  int reduce_m1 = 0, reduce_m2 = 0; // chunk sizes of the two levels (0 = 8 and 4), tuning aid
  int pair_variant = 0; // launch-bound variant / code layout of the pairing kernels (tuning aid); >= 16: Miller and final exponentiation as two kernels
  int coop_max_n = 10240;           // batches of at most this many BLS12-381 pairings / checks run one per WARP (coop_pairing.cuh; near the measured
                                    // break-even with the one-per-thread kernels); 0 = never
  void* pair_scratch = nullptr;     // Miller values between the two kernels of the split pairing (576 B per element; grown on demand)
  size_t pair_scratch_cap = 0;
  int msm_layout = 0;   // 0 = compact field products (library default), 1 = inlined at every use (b2k_msm_inlined.cu): A/B aid
  int last_plan[LP_SLOTS] = {};     // what the last MSM ran with (MsmPlanSlot)
  uint64_t launches = 0;
  std::string err;
};

// scratch arena (defined in b2k_api.cu): reserve resets the arena and grows it if needed;
// take returns 256-byte aligned sub-buffers or nullptr.  A call reserves it at most once, through arena_carve, host_call or
// msm_begin (host_call.cuh, msm_host.cuh), so nothing it has taken is handed out again while the call runs.
int b2k_arena_reserve(b2k_ctx* ctx, size_t bytes);
void* b2k_arena_take(b2k_ctx* ctx, size_t bytes);

// internal entry points shared between translation units (not part of include/b2kyber.h)
extern "C" int b2k_internal_bls12381_g1_msm_buckets_host(b2k_ctx* c, size_t n, const uint8_t* s, const uint8_t* p, void* b, size_t cap, int* plan);
extern "C" int b2k_internal_bls12381_g1_msm_dev_inlined(b2k_ctx* c, size_t n, const void* s, const void* p, void* o, int affine_out);
extern "C" int b2k_internal_bls12381_g1_mul_batch_dev_inlined(b2k_ctx* c, size_t n, const void* s, const void* p, void* o, int affine_out);
