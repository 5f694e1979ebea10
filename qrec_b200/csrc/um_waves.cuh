// The wave schedule of the user-major BPR epoch (bpr_kernels.cu: launch_usermajor), for host and device.
//
// The n triples of one launch (CSR order over users; rowptr holds GLOBAL triple offsets, the launch's
// triples are [trip_off, trip_off + n)) are cut into chunks of UM_CH triples and the chunks are swept in
// waves of um_wave_chunks() chunks.  Before a wave the item table is snapshotted, and the wave reads item
// rows only from that snapshot.  A user belongs to the wave whose chunks hold its first triple and is
// processed whole there, even where it runs on into later waves' chunks; the launch's first user starts at
// the launch's first triple and its last user ends at its last, wherever the caller cut them.  Users with no
// triples belong to no wave.
//
// So wave w is the users [um_wave_first_user(w), um_wave_first_user(w + 1)).
#pragma once

#if defined(__CUDACC__)
#define QREC_HD __host__ __device__
#else
#define QREC_HD
#endif

namespace qrec {

constexpr int UM_CH = 32;   // triples per chunk: wave boundaries fall on multiples of UM_CH

// Wave length in chunks for a launch of n triples on an item table of num_items rows of width d (fp32).
// No more than 4 x the item rows, so an item row is read only a few of its own updates late.  On a small table
// (snapshot copy under 8 MB, about the cost of a launch) at least 64 waves per launch: on a small data set the hot
// items recur within a few hundred triples.  On a large one the wave is long enough that the copy stays under 1/8
// of the wave's algorithmic bytes (24 d + 12 per triple).
QREC_HD inline long long um_wave_chunks(long long n, long long num_items, int d) {
  const long long copy_bytes = 2 * num_items * d * 4;
  const long long copy_floor = copy_bytes > (8LL << 20) ? 8 * copy_bytes / (24LL * d + 12) : 0;
  long long wave_triples = n / 64 > copy_floor ? n / 64 : copy_floor;
  if (wave_triples > 4 * num_items) wave_triples = 4 * num_items;
  return wave_triples / UM_CH > 1 ? wave_triples / UM_CH : 1;
}

QREC_HD inline long long um_num_waves(long long n, long long wave_chunks) {
  const long long nchunks = (n + UM_CH - 1) / UM_CH;
  return (nchunks + wave_chunks - 1) / wave_chunks;
}

// First user of wave w (w = um_num_waves() gives one past the launch's last user).  Wave 0 starts with the user of
// the launch's first triple: the smallest u with rowptr[u + 1] > trip_off.  A later wave starts with the first user
// whose first triple is at or after the wave's first triple b: the smallest u with rowptr[u] >= trip_off + b.
QREC_HD inline int um_wave_first_user(const long long* rowptr, int n_users, long long n, long long trip_off,
                                      long long wave_chunks, long long w) {
  long long b = w * wave_chunks * UM_CH;
  if (b > n) b = n;
  const long long key = b == 0 ? trip_off + 1 : trip_off + b;
  const long long* a = b == 0 ? rowptr + 1 : rowptr;
  int lo = 0, hi = b == 0 ? n_users : n_users + 1;   // answer in [lo, hi]; hi means "none"
  while (lo < hi) {
    const int mid = lo + (hi - lo) / 2;
    if (a[mid] >= key) hi = mid;
    else lo = mid + 1;
  }
  return lo;
}

}  // namespace qrec
