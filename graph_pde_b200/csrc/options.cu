#include "options.h"

#include <cstdlib>
#include <cstring>
#include <mutex>

namespace nnc {

namespace {
using Field = int Options::*;
struct Entry {
  const char* name;       // option name == environment variable without the NNCONV_ prefix, lower case
  const char* env;
  Field field;
  int dflt;
};
const Entry kEntries[] = {
    {"no_fuse", "NNCONV_NO_FUSE", &Options::no_fuse, 0},
    {"no_pipe", "NNCONV_NO_PIPE", &Options::no_pipe, 0},
    {"ring", "NNCONV_RING", &Options::ring, 3},
    {"ring_deep", "NNCONV_RING_DEEP", &Options::ring_deep, 0},
    {"apply_stages", "NNCONV_APPLY_STAGES", &Options::apply_stages, 0},
    {"apply_passes", "NNCONV_APPLY_PASSES", &Options::apply_passes, 0},
    {"apply_a_policy", "NNCONV_APPLY_A_POLICY", &Options::apply_a_policy, 0},
    {"tmap_promo", "NNCONV_TMAP_PROMO", &Options::tmap_promo, 2},
    {"scatter_mode", "NNCONV_SCATTER_MODE", &Options::scatter_mode, 1},
    {"debug_scatter", "NNCONV_DEBUG_SCATTER", &Options::debug_scatter, 0},
    {"y_store_policy", "NNCONV_Y_STORE_POLICY", &Options::y_store_policy, 0},
    {"l2_persist", "NNCONV_L2_PERSIST", &Options::l2_persist, 0},
    {"l2_reset", "NNCONV_L2_RESET", &Options::l2_reset, 0},
    {"gemm_b_policy", "NNCONV_GEMM_B_POLICY", &Options::gemm_b_policy, 1},
    {"conv_one_per_sm", "NNCONV_CONV_ONE_PER_SM", &Options::conv_one_per_sm, 0},
    {"conv_stages", "NNCONV_CONV_STAGES", &Options::conv_stages, 0},
    {"conv_debug", "NNCONV_DEBUG", &Options::conv_debug, 0},
    {"gemm_direct_store", "NNCONV_GEMM_DIRECT_STORE", &Options::gemm_direct_store, 0},
    {"trace", "NNCONV_TRACE", &Options::trace, 0},
    {"no_coop", "NNCONV_NO_COOP", &Options::no_coop, 0},
    {"overflow_check", "NNCONV_OVERFLOW_CHECK", &Options::overflow_check, 1},
};
Options g_opt;
std::once_flag g_once;

void sanitize(Options& o) {
  if (o.ring < 2 || o.ring > 8) o.ring = 3;
}
}  // namespace

Options& options() {
  std::call_once(g_once, [] {
    for (const Entry& e : kEntries) {
      const char* v = getenv(e.env);
      // a variable that is set but empty or non-numeric counts as "1" (the historical `NNCONV_NO_FUSE=` usage)
      g_opt.*(e.field) = v == nullptr ? e.dflt : ((*v >= '0' && *v <= '9') || *v == '-') ? atoi(v) : 1;
    }
    sanitize(g_opt);
  });
  return g_opt;
}

int option_set(const char* name, int value) {
  Options& o = options();
  for (const Entry& e : kEntries) {
    if (strcmp(e.name, name) == 0) {
      o.*(e.field) = value < -1000000 ? e.dflt : value;   // value < -1e6: restore the built-in default
      sanitize(o);
      return 0;
    }
  }
  return -1;
}

int option_get(const char* name, int* value) {
  Options& o = options();
  for (const Entry& e : kEntries) {
    if (strcmp(e.name, name) == 0) {
      *value = o.*(e.field);
      return 0;
    }
  }
  return -1;
}

}  // namespace nnc
