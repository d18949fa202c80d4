// Error reporting / bookkeeping shared by all entry points.
#include <atomic>
#include <cstdarg>
#include <cstdio>
#include <cstdlib>

#include "sq_common.cuh"

namespace sq {
static thread_local char g_err[512] = "";
std::atomic<uint64_t> g_launches{0};

void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}
bool pdl_enabled() {
  static int v = -1;
  if (v < 0) {
    const char* e = getenv("SQ_PDL");           // programmatic dependent launch: on by default, SQ_PDL=0 turns it off
    v = (e && !atoi(e)) ? 0 : 1;
  }
  return v == 1;
}
void count_launch(int n) { g_launches.fetch_add((uint64_t)n, std::memory_order_relaxed); }

int make_ragged(const sq_ragged_part* parts, int n_parts, int B, int n_max, int rows_per_tile, const char* who,
                RaggedParts* out) {
  SQ_CHECK_ARG(parts != nullptr && B >= 1 && B <= SQ_MAX_BATCH && rows_per_tile >= 1, "%s: null parts or B=%d (1..%d)",
               who, B, SQ_MAX_BATCH);
  SQ_CHECK_ARG(n_parts >= 1 && n_parts <= B, "%s: %d parts for %d sequences", who, n_parts, B);
  *out = RaggedParts{};
  out->n_parts = n_parts;
  unsigned seen = 0;
  int64_t rows = 0, tiles = 0;
  for (int j = 0; j < n_parts; ++j) {
    const sq_ragged_part& p = parts[j];
    SQ_CHECK_ARG(p.seq >= 0 && p.seq < B, "%s: part %d names sequence %d of %d", who, j, p.seq, B);
    SQ_CHECK_ARG(!(seen >> p.seq & 1u), "%s: sequence %d listed twice", who, p.seq);
    SQ_CHECK_ARG(p.n >= 1, "%s: part %d has n=%d rows", who, j, p.n);
    seen |= 1u << p.seq;
    out->seq[j] = p.seq; out->n[j] = p.n; out->n0[j] = p.n0; out->kv_end[j] = p.kv_end;
    out->row0[j] = (int)rows;
    out->tile0[j] = (int)tiles;
    rows += p.n;
    tiles += (p.n + rows_per_tile - 1) / rows_per_tile;
    SQ_CHECK_ARG(rows <= n_max, "%s: %lld rows exceed n_max=%d", who, (long long)rows, n_max);
  }
  out->row0[n_parts] = (int)rows;
  out->tile0[n_parts] = (int)tiles;
  return SQ_OK;
}
}  // namespace sq

extern "C" int sq_ragged_layout(const sq_ragged_part* parts, int n_parts, int B, int n_max, int rows_per_tile,
                                int32_t* row0, int32_t* tile0) {
  sq::RaggedParts rp;
  const int rc = sq::make_ragged(parts, n_parts, B, n_max, rows_per_tile, "sq_ragged_layout", &rp);
  if (rc != SQ_OK) return rc;
  for (int j = 0; j <= n_parts; ++j) {
    if (row0) row0[j] = rp.row0[j];
    if (tile0) tile0[j] = rp.tile0[j];
  }
  return SQ_OK;
}

extern "C" const char* sq_last_error(void) { return sq::g_err; }
extern "C" int sq_version(void) { return 100; }
extern "C" uint64_t sq_launch_count(void) { return sq::g_launches.load(std::memory_order_relaxed); }
