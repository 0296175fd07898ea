// Minimum-Bayes-risk selection (fira_icse_b200/mbr.py, fira_mbr_select): per commit, the sample with the highest mean
// sentence BLEU against the commit's other samples.  The rule is stated in include/fira_b200.h.
//
// One CTA per commit, everything in shared memory:
//   compact   warp n cleans candidate n (drops start / eos / pad ids from columns 1..length-1) with a ballot
//   matches   for candidates a (hypothesis side) and b, lane p of a warp builds the bit mask over b's positions q
//             where the n-gram of a starting at p occurs: bit q of E_p = (b[q] == a[p]) comes from one ballot per p
//             (lane q holds b[q]), and the orders follow by shifts of the neighbours' masks,
//             M1 = E_p, M2 = M1 & (E_p+1 >> 1), M3 = M2 & (E_p+2 >> 2), M4 = M3 & (E_p+3 >> 3)
//   counts    a = b = i: lane p keeps c_i = popc(M) when no lower bit is set (the n-gram occurs first at p), else 0
//   pairs     one warp per unordered pair i <= j (a = i, b = j).  Clipped matches sum_g min(c_i(g), c_j(g)) are
//             symmetric in i and j, so the four warp sums of min(c_i, popc(M)) are the numerators of both BLEU(i, j)
//             and BLEU(j, i)
//   scores    one thread per ordered pair evaluates BLEU in float64 into the N x N shared matrix; thread i sums row i
//             in ascending j; thread 0 takes the first maximum
// Bounded by the pair pass: N(N+1)/2 warps of one ballot per word of i (at most 528 x 31 at N = 32).
#include "common.cuh"

namespace {

constexpr int kMbrThreads = 512;
constexpr int kMbrWarps = kMbrThreads / kWarp;
constexpr int kMaxCand = 32;          // sample.MAX_SAMPLES
constexpr int kMaxT = 32;             // T_len: at most 31 words per candidate, one per lane

// sentence_bleu_method2([ref], hyp) from the clipped match counts num[n] of orders n + 1, c = len(hyp), r = len(ref);
// the same operation order as fira_icse_b200/bleu.py (explicit roundings: no fused multiply-add)
__device__ double method2_bleu(const int (&num)[4], int c, int r) {
  if (c == 0 || num[0] == 0) return 0.0;
  double logs = 0.0;
#pragma unroll
  for (int n = 0; n < 4; ++n) {
    const int den = max(1, c - n);
    const double q = n == 0 ? (double)num[0] / (double)den : (double)(num[n] + 1) / (double)(den + 1);
    logs = __dadd_rn(logs, __dmul_rn(0.25, log(q)));
  }
  const double bp = c > r ? 1.0 : exp(1.0 - (double)r / (double)c);
  return __dmul_rn(bp, exp(logs));
}

// M[n] of this lane (p = lane): bit q set when the n + 1 words of `a` from p equal those of `b` from q.  Valid for
// p + n < la; lanes at or past the end of `a` get garbage the callers mask.
__device__ __forceinline__ void match_masks(const int* a, int la, const int* b, int lb, int lane, unsigned (&M)[4]) {
  const int mine = b[lane];
  unsigned e = 0;
  for (int p = 0; p < la; ++p) {
    const unsigned bits = __ballot_sync(0xffffffffu, lane < lb && mine == a[p]);
    if (lane == p) e = bits;
  }
  M[0] = e;
  M[1] = M[0] & (__shfl_down_sync(0xffffffffu, e, 1) >> 1);
  M[2] = M[1] & (__shfl_down_sync(0xffffffffu, e, 2) >> 2);
  M[3] = M[2] & (__shfl_down_sync(0xffffffffu, e, 3) >> 3);
}

__global__ void __launch_bounds__(kMbrThreads) mbr_select_kernel(
    const int* __restrict__ seq, const int* __restrict__ length, long ld_seq, int start_id, int eos_id, int pad_id,
    double* __restrict__ pair_bleu, double* __restrict__ utility, int* __restrict__ best, int N, int T_len) {
  pdl_wait(); pdl_trigger();       // PDL (common.cuh)
  __shared__ int s_words[kMaxCand][kWarp];
  __shared__ int s_len[kMaxCand];
  __shared__ unsigned char s_cnt[kMaxCand][4][kWarp];   // c_i of the n-gram starting at p if it occurs first there
  __shared__ unsigned s_num[kMaxCand * kMaxCand];       // [i * N + j] = the four numerators, 8 bits each (<= 31)
  __shared__ double s_pair[kMaxCand * kMaxCand];        // [i * N + j] = BLEU(i, j)
  __shared__ double s_util[kMaxCand];
  const int b = blockIdx.x, warp = threadIdx.x / kWarp, lane = threadIdx.x % kWarp;

  for (int n = warp; n < N; n += kMbrWarps) {
    const long row = (long)b * N + n;
    const int L = min(max(length[row], 1), T_len);
    const int col = 1 + lane;
    int id = 0;
    bool keep = false;
    if (col < L) {
      id = seq[row * ld_seq + col];
      keep = id != start_id && id != eos_id && id != pad_id;
    }
    const unsigned ballot = __ballot_sync(0xffffffffu, keep);
    if (keep) s_words[n][__popc(ballot & ((1u << lane) - 1u))] = id;
    if (lane == 0) s_len[n] = __popc(ballot);
  }
  __syncthreads();

  for (int i = warp; i < N; i += kMbrWarps) {
    unsigned M[4];
    match_masks(s_words[i], s_len[i], s_words[i], s_len[i], lane, M);
    const unsigned below = (1u << lane) - 1u;
#pragma unroll
    for (int n = 0; n < 4; ++n)
      s_cnt[i][n][lane] = (lane + n < s_len[i] && (M[n] & below) == 0) ? (unsigned char)__popc(M[n]) : 0;
  }
  __syncthreads();

  for (int e = warp; e < N * N; e += kMbrWarps) {
    const int i = e / N, j = e % N;
    if (j < i) continue;
    unsigned M[4];
    match_masks(s_words[i], s_len[i], s_words[j], s_len[j], lane, M);
    unsigned packed = 0;
#pragma unroll
    for (int n = 0; n < 4; ++n)
      packed |= __reduce_add_sync(0xffffffffu, min((unsigned)s_cnt[i][n][lane], (unsigned)__popc(M[n]))) << (8 * n);
    if (lane == 0) { s_num[i * N + j] = packed; s_num[j * N + i] = packed; }
  }
  __syncthreads();

  for (int e = threadIdx.x; e < N * N; e += kMbrThreads) {
    const int i = e / N, j = e % N;
    const unsigned packed = s_num[e];
    const int num[4] = {(int)(packed & 0xFFu), (int)((packed >> 8) & 0xFFu), (int)((packed >> 16) & 0xFFu),
                        (int)(packed >> 24)};
    s_pair[e] = method2_bleu(num, s_len[i], s_len[j]);
  }
  __syncthreads();

  if (threadIdx.x < N) {
    const int i = threadIdx.x;
    double sum = 0.0;
    for (int j = 0; j < N; ++j)
      if (j != i) sum += s_pair[i * N + j];
    s_util[i] = sum / (double)(N - 1);
    utility[(long)b * N + i] = s_util[i];
  }
  if (pair_bleu)
    for (int e = threadIdx.x; e < N * N; e += kMbrThreads) pair_bleu[(long)b * N * N + e] = s_pair[e];
  __syncthreads();
  if (threadIdx.x == 0) {
    int arg = 0;
    for (int i = 1; i < N; ++i)
      if (s_util[i] > s_util[arg]) arg = i;
    best[b] = arg;
  }
}

// Self-critical rewards (fira_icse_b200/scst.py, fira_bleu_reward): per commit, the sentence BLEU of each sample against
// the commit's reference and its leave-one-out advantage.  One CTA per commit, one warp per sample:
//   reference  warp 0 cleans ref columns 1..T_len-1 before the first eos_id (start / pad ids dropped) into shared memory
//   sample     warp n cleans sample n as fira_mbr_select does, then lane p keeps c_p = the count of the sample's n-gram at
//              p where it occurs first (match_masks of the sample against itself) and the warp sums min(c_p, occurrences
//              in the reference) per order: the clipped matches of sentence_bleu_method2([ref], sample)
//   baseline   thread n: A_n = (sum over m != n, m ascending, of (r_n - r_m)) / (N - 1): exactly 0 when the rewards tie
__global__ void __launch_bounds__(kMaxCand * kWarp) bleu_reward_kernel(
    const int* __restrict__ seq, const int* __restrict__ length, long ld_seq, const int* __restrict__ ref, long ld_ref,
    int start_id, int eos_id, int pad_id, double* __restrict__ reward, double* __restrict__ advantage, int N, int T_len) {
  pdl_wait(); pdl_trigger();       // PDL (common.cuh)
  __shared__ int s_ref[kWarp];
  __shared__ int s_ref_len;
  __shared__ int s_words[kMaxCand][kWarp];
  __shared__ double s_r[kMaxCand];
  const int b = blockIdx.x, n = threadIdx.x / kWarp, lane = threadIdx.x % kWarp;
  const int col = 1 + lane;

  if (n == 0) {
    const int id = col < T_len ? ref[(long)b * ld_ref + col] : eos_id;
    const unsigned eos = __ballot_sync(0xffffffffu, id == eos_id);    // lane 31 (col = T_len at most) always votes
    const bool keep = lane < __ffs(eos) - 1 && id != start_id && id != pad_id;
    const unsigned ballot = __ballot_sync(0xffffffffu, keep);
    if (keep) s_ref[__popc(ballot & ((1u << lane) - 1u))] = id;
    if (lane == 0) s_ref_len = __popc(ballot);
  }
  const long row = (long)b * N + n;
  const int L = min(max(length[row], 1), T_len);
  int id = 0;
  bool keep = false;
  if (col < L) {
    id = seq[row * ld_seq + col];
    keep = id != start_id && id != eos_id && id != pad_id;
  }
  const unsigned ballot = __ballot_sync(0xffffffffu, keep);
  if (keep) s_words[n][__popc(ballot & ((1u << lane) - 1u))] = id;
  const int c = __popc(ballot);
  __syncthreads();

  unsigned M[4];
  match_masks(s_words[n], c, s_words[n], c, lane, M);
  const unsigned below = (1u << lane) - 1u;
  unsigned cnt[4];
#pragma unroll
  for (int k = 0; k < 4; ++k) cnt[k] = (lane + k < c && (M[k] & below) == 0) ? __popc(M[k]) : 0u;
  match_masks(s_words[n], c, s_ref, s_ref_len, lane, M);
  int num[4];
#pragma unroll
  for (int k = 0; k < 4; ++k) num[k] = (int)__reduce_add_sync(0xffffffffu, min(cnt[k], (unsigned)__popc(M[k])));
  if (lane == 0) {
    s_r[n] = method2_bleu(num, c, s_ref_len);
    reward[row] = s_r[n];
  }
  __syncthreads();

  if (threadIdx.x < N) {
    const int i = threadIdx.x;
    double sum = 0.0;
    for (int m = 0; m < N; ++m)
      if (m != i) sum = __dadd_rn(sum, __dsub_rn(s_r[i], s_r[m]));
    advantage[(long)b * N + i] = sum / (double)(N - 1);
  }
}

}  // namespace

extern "C" int fira_bleu_reward(const int* seq, const int* length, long ld_seq, const int* ref, long ld_ref,
                                int start_id, int eos_id, int pad_id, double* reward, double* advantage, int B, int N,
                                int T_len, void* stream) {
  FIRA_CHECK_ARG(B >= 0 && N >= 2 && N <= kMaxCand, FIRA_ERR_SHAPE, "bleu_reward: B %d, N %d (2 <= N <= %d)", B, N,
                 kMaxCand);
  FIRA_CHECK_ARG(T_len >= 2 && T_len <= kMaxT && ld_seq >= T_len && ld_ref >= T_len, FIRA_ERR_SHAPE,
                 "bleu_reward: T_len %d, ld_seq %ld, ld_ref %ld (2 <= T_len <= %d, ld_seq, ld_ref >= T_len)", T_len,
                 ld_seq, ld_ref, kMaxT);
  if (B == 0) return FIRA_OK;
  FIRA_CHECK_ARG(seq && length && ref && reward && advantage, FIRA_ERR_ARG,
                 "bleu_reward: null seq / length / ref / reward / advantage");
  launch_k(bleu_reward_kernel, dim3((unsigned)B), dim3((unsigned)(N * kWarp)), 0, (cudaStream_t)stream, seq, length,
           ld_seq, ref, ld_ref, start_id, eos_id, pad_id, reward, advantage, N, T_len);
  FIRA_CHECK_LAUNCH("fira_bleu_reward");
  return FIRA_OK;
}

extern "C" int fira_mbr_select(const int* seq, const int* length, long ld_seq, int start_id, int eos_id, int pad_id,
                               double* pair_bleu, double* utility, int* best, int B, int N, int T_len, void* stream) {
  FIRA_CHECK_ARG(B >= 0 && N >= 2 && N <= kMaxCand, FIRA_ERR_SHAPE, "mbr_select: B %d, N %d (2 <= N <= %d)", B, N,
                 kMaxCand);
  FIRA_CHECK_ARG(T_len >= 2 && T_len <= kMaxT && ld_seq >= T_len, FIRA_ERR_SHAPE,
                 "mbr_select: T_len %d, ld_seq %ld (2 <= T_len <= %d, ld_seq >= T_len)", T_len, ld_seq, kMaxT);
  if (B == 0) return FIRA_OK;
  FIRA_CHECK_ARG(seq && length && utility && best, FIRA_ERR_ARG, "mbr_select: null seq / length / utility / best");
  launch_k(mbr_select_kernel, dim3((unsigned)B), dim3(kMbrThreads), 0, (cudaStream_t)stream, seq, length, ld_seq,
           start_id, eos_id, pad_id, pair_bleu, utility, best, N, T_len);
  FIRA_CHECK_LAUNCH("fira_mbr_select");
  return FIRA_OK;
}
