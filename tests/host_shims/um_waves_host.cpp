// Host build of qrec_b200/csrc/um_waves.cuh: the wave schedule of the user-major BPR epoch, so that the CPU suite
// can check the wave table launch_usermajor computes on the device against the chunk rule it restates.
#include "um_waves.cuh"

extern "C" {

long long um_wave_chunks_host(long long n, long long num_items, int d) { return qrec::um_wave_chunks(n, num_items, d); }

// wave_user[0 .. nwaves] as um_wave_table_kernel writes it; returns nwaves, or -1 if `cap` entries do not suffice
long long um_wave_table_host(const long long* rowptr, int n_users, long long n, long long trip_off, long long num_items, int d,
                             int* wave_user, long long cap) {
  const long long wave = qrec::um_wave_chunks(n, num_items, d);
  const long long nwaves = qrec::um_num_waves(n, wave);
  if (nwaves + 1 > cap) return -1;
  for (long long w = 0; w <= nwaves; ++w) wave_user[w] = qrec::um_wave_first_user(rowptr, n_users, n, trip_off, wave, w);
  return nwaves;
}

}  // extern "C"
