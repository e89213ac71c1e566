// Exhaustive host-side check of the stream-K partition arithmetic (substratus_b200/csrc/sk_partition.h) that
// tc_gemm_sk_kernel and its launcher use: for every projection shape of the BASELINE models (full and tensor-parallel
// shards), a sweep of odd shapes and several SM counts, rebuild the segment structure by brute force and compare with what
// an owner CTA computes for itself.  Prints "OK <cases>" or the first violation.  Built and run by tests/test_sk_partition_cpu.py.
#include <cstdio>
#include <cstdlib>
#include <vector>

#include "../substratus_b200/csrc/sk_partition.h"

struct Seg {
  int cta, tile, kb0, kb1;
  bool first;
};

static int check(long long N, long long K, int n_sm) {
  const int nkb = (int)((K + 63) / 64), n_ntiles = (int)((N + 127) / 128);
  const long long Ull = (long long)n_ntiles * nkb;
  const int G = sk_grid(Ull, nkb, n_sm);
  if (!sk_fits(Ull, G)) return 0;  // the launcher refuses (cudaErrorInvalidValue); nothing to check
  const int U = (int)Ull;
  if (G < 1 || G > n_sm || G > U) return printf("N %lld K %lld sm %d: bad grid %d (U %d)\n", N, K, n_sm, G, U), 1;
  std::vector<Seg> segs;
  std::vector<int> owner(n_ntiles, -1), owner_end(n_ntiles, 0);
  std::vector<std::vector<int>> contrib(n_ntiles);
  int prev_end = 0;
  for (int b = 0; b < G; ++b) {
    const int u0 = sk_begin(b, U, G), u1 = sk_begin(b + 1, U, G);
    if (u0 != prev_end || u1 <= u0) return printf("N %lld K %lld sm %d: range of CTA %d is [%d, %d) after %d\n", N, K, n_sm, b, u0, u1, prev_end), 1;
    prev_end = u1;
    for (int u = u0; u < u1;) {  // the kernel's own segment walk
      const int nt = u / nkb, kb0 = u - nt * nkb;
      const int kb1 = nkb < kb0 + (u1 - u) ? nkb : kb0 + (u1 - u);
      if (kb0 != 0) {
        if (u != u0) return printf("N %lld K %lld sm %d: CTA %d has a contributor segment that is not its first\n", N, K, n_sm, b), 1;
        contrib[nt].push_back(b);
      } else {
        if (owner[nt] != -1) return printf("N %lld K %lld sm %d: tile %d has two owners\n", N, K, n_sm, nt), 1;
        owner[nt] = b;
        owner_end[nt] = u + (kb1 - kb0);
      }
      u += kb1 - kb0;
    }
  }
  if (prev_end != U) return printf("N %lld K %lld sm %d: ranges end at %d, U = %d\n", N, K, n_sm, prev_end, U), 1;
  for (int nt = 0; nt < n_ntiles; ++nt) {
    const int b = owner[nt];
    if (b < 0) return printf("N %lld K %lld sm %d: tile %d has no owner\n", N, K, n_sm, nt), 1;
    const int n = sk_contributors(b, U, G, owner_end[nt], (nt + 1) * nkb);
    if (n != (int)contrib[nt].size() || n > 10)
      return printf("N %lld K %lld sm %d: tile %d owner %d counts %d contributors, there are %zu\n", N, K, n_sm, nt, b, n, contrib[nt].size()), 1;
    for (int i = 0; i < n; ++i)  // the owner reads slots 2 (b + 1 + i): they must be exactly the contributors, all later CTAs
      if (contrib[nt][i] != b + 1 + i || 2 * (b + 1 + i) + 1 >= 2 * G + 2)
        return printf("N %lld K %lld sm %d: tile %d contributor %d is CTA %d, owner %d expects %d\n", N, K, n_sm, nt, i, contrib[nt][i], b, b + 1 + i), 1;
  }
  return 0;
}

int main() {
  long long cases = 0;
  const int sms[] = {148, 147, 132, 108, 64, 17, 8, 2, 1};
  // (rows N, reduction K) of q|k|v, o, gate|up, down, lm_head at hidden / intermediate / heads of the BASELINE models
  struct M { long long h, inter, q_rows, kv_rows, vocab; };
  const M models[] = {{4096, 11008, 4096, 4096, 32000}, {5120, 13824, 5120, 5120, 32000}, {8192, 28672, 8192, 1024, 32000},
                      {768, 3072, 768, 768, 50272}, {2048, 2816, 2048, 1024, 1008}, {8192, 32768, 8192, 1024, 65024}};
  for (const M& m : models)
    for (int tp : {1, 2, 4, 8}) {
      const long long shapes[][2] = {{(m.q_rows + 2 * m.kv_rows) / tp, m.h}, {m.h, m.q_rows / tp}, {2 * m.inter / tp, m.h},
                                     {m.h, m.inter / tp}, {m.vocab, m.h}};
      for (auto& s : shapes)
        for (int sm : sms) {
          if (s[0] < 2 || s[1] < 8) continue;
          if (check(s[0], s[1], sm)) return 1;
          ++cases;
        }
    }
  // odd shapes: every tile count up to 40 x k-block counts around the grid size, ragged N and K
  for (long long nt = 1; nt <= 40; ++nt)
    for (long long kb = 1; kb <= 200; kb += (kb < 20 ? 1 : 7))
      for (int sm : sms) {
        if (check(nt * 128 - (nt % 3) * 2, kb * 64 - (kb % 2) * 8, sm)) return 1;
        ++cases;
      }
  // large: vocab 256k x hidden 16k stays inside the 32-bit arithmetic
  if (check(256000, 16384, 132)) return 1;
  ++cases;
  printf("OK %lld\n", cases);
  return 0;
}
