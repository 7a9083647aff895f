// Tuning / debugging knobs of libnnconv_b200.  They are read from the environment ONCE (first nnconv_init)
// and can afterwards be changed through nnconv_set_option(); nothing on the per-application path calls getenv.
#pragma once

namespace nnc {

struct Options {
  int no_fuse;            // NNCONV_NO_FUSE: per-batch Y GEMM + contraction kernels instead of the persistent fused kernel
  int no_pipe;            // NNCONV_NO_PIPE: plain stream order for the per-batch kernels (no PDL / flags)
  int ring;               // NNCONV_RING: Y ring depth of the fused kernel (2..8, default 3)
  int ring_deep;          // NNCONV_RING_DEEP (default 0): when the Y budget holds more than ring x 128 sources (narrow edge
                          // networks: 32 KB of Y per source at ker_width 256), keep batches of 128 sources and deepen the
                          // ring (<= 16) instead of growing the batches; off by default: more batches = more flag round
                          // trips per launch
  int apply_stages;       // NNCONV_APPLY_STAGES: cap on the A stages of the fused kernel (0 = no cap)
  int apply_passes;       // NNCONV_APPLY_PASSES: force the number of passes over the B-slot ring (0 = automatic): more
                          // passes = fewer resident B slots = more A stages (bytes of the h stream in flight)
  int apply_a_policy;     // NNCONV_APPLY_A_POLICY: L2 hint of the h stream in the fused kernel: 0 evict-first (default), 1 normal
  int tmap_promo;         // NNCONV_TMAP_PROMO: L2 promotion of operand tensor maps: 2 = 256 B (default), 1 = 128 B, 0 = none
  int scatter_mode;       // NNCONV_SCATTER_MODE: 1 (default) = each edge row staged in shared memory and added to out[dst] with
                          // ONE cp.reduce.async.bulk (256 B per request, TMA engine); 0 = red.global.add.v2.f32 straight
                          // from the accumulator fragments (8 B per request)
  int debug_scatter;      // NNCONV_DEBUG_SCATTER: timing experiments only (wrong results)
  int y_store_policy;     // NNCONV_Y_STORE_POLICY: 0 normal, 1 evict-last, 2 evict-first
  int l2_persist;         // NNCONV_L2_PERSIST: access-policy window over the Y ring; value = persisting-L2 set-aside in MB
                          // (1 = the device maximum)
  int l2_reset;           // NNCONV_L2_RESET: cudaCtxResetPersistingL2Cache at the start of every edge-feature pass
  int gemm_b_policy;      // NNCONV_GEMM_B_POLICY: L2 hint of the GEMM's B (weight) tiles: 1 evict-last (default), 0 normal
  int conv_one_per_sm;    // NNCONV_CONV_ONE_PER_SM
  int conv_stages;        // NNCONV_CONV_STAGES
  int conv_debug;         // NNCONV_DEBUG
  int gemm_direct_store;  // NNCONV_GEMM_DIRECT_STORE: st.global epilogue instead of TMA stores
  int trace;              // NNCONV_TRACE: CTA timeline records
  int no_coop;            // NNCONV_NO_COOP: launch the fused kernel without the cooperative attribute
  int overflow_check;     // NNCONV_OVERFLOW_CHECK: count non-finite / saturated 16-bit edge features (default 1)
};

Options& options();                          // initialised from the environment on first use
int option_set(const char* name, int value); // 0 ok, -1 unknown name
int option_get(const char* name, int* value);

}  // namespace nnc
