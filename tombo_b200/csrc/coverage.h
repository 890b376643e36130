// coverage.h -- the project's one coverage builder (defined in read_filter.cu), shared by
// tb2_read_mid_coverage and tb2_coverage_runs: every (chromosome, strand) group's read
// coverage from a difference array and one device-wide prefix sum (read_filter.cuh).
#pragma once
#include "ctx.h"
#include <vector>

// the caller's workspace, five consecutive DevBufs in this order
enum { COV_START = 0, COV_END, COV_DIFF, COV_TSUM, COV_TOFF, COV_BUFS };

// Reads of group g are grp_off[g] .. grp_off[g + 1] (grp_off[0] = 0 and non-decreasing, checked
// by the caller).  Checks 0 <= start < end for every read ("<what>: every read needs 0 <= start
// < end"), then places the groups one after another: a group with reads takes max(end) + 1
// entries from base[g] (the last entry takes the -1 of the reads that end there), an empty group
// none; base[n_groups] is the total length.  Uploads the absolute starts and ends to
// ws[COV_START] / ws[COV_END] (long long), records ctx->ev0 (kernel time starts here) and leaves
// the coverage, int per entry, in ws[COV_DIFF].  Enqueued on ctx->stream, not synchronised.
int tb2_coverage_build(tb2_ctx *ctx, const char *what, DevBuf *ws, int64_t n_groups, const int64_t *grp_off,
                       const int64_t *start, const int64_t *end, std::vector<long long> &base);

// inclusive prefix sum of x[0 .. len) in place (int entries, long long partial sums), with
// ws[COV_TSUM] / ws[COV_TOFF] as the tiles' scratch: the scan inside tb2_coverage_build.
// Enqueued on ctx->stream.
int tb2_coverage_scan(tb2_ctx *ctx, const char *what, DevBuf *ws, int *x, long long len);
