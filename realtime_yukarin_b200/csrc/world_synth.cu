// world_synth.cu -- WORLD realtime synthesizer on the H100 (SURVEY row a14, component J).
// Replaces world4py's _InitializeSynthesizer / _AddParameters / _Synthesis2 (call sites:
// realtime_voice_conversion/yukarin_wrapper/vocoder.py:79-103) with a device-resident state machine:
//   k_synth_add     one CTA : append frames to the device ring, sample-rate f0/vuv interpolation,
//                             total-phase prefix scan (FP64 block scan), ordered pulse compaction
//   k_synth_noise   one CTA : xorshift128 randn stream, addressed by absolute sample position,
//                             generated in 8192-position tiles with GF(2) jump-ahead matrices
//   k_synth_plan    one warp: how many 1024-sample blocks may be emitted + which pulses they need
//   k_synth_pulse   one CTA per pulse: spectral/aperiodic interpolation, 2 minimum-phase
//                             reconstructions + noise FFT + 2 inverse FFTs, all in shared memory
//   k_synth_ola     gather-style overlap-add in pulse order (deterministic), emits blocks + new carry
// The state (frame ring, pulse ring, noise ring, OLA carry, hand-off phase/f0) never leaves HBM.
#include <math.h>
#include <string.h>
#include <vector>

#include "engine.h"
#include "fft.cuh"
#include "synth.h"

namespace ryk {

__device__ inline double safe_ap(double x) { return fmax(0.001, fmin(0.999999999999, x)); }

// ------------------------------------------------------------------------------------ add parameters
__global__ void __launch_bounds__(1024) k_synth_add(SynthDev S, const double* __restrict__ f0, int n,
                                                   const float* __restrict__ sp, const float* __restrict__ ap) {
  SynthState* st = S.state;
  __shared__ double scan_scratch[1024];
  __shared__ long long sh_first_frame, sh_start;
  __shared__ int sh_ns, sh_hf, sh_ok;
  __shared__ double sh_handoff_f0;
  __shared__ int wsum[32];
  __shared__ int sh_total;
  const int nb = S.fft_size / 2 + 1;
  const double fp = S.frame_period, fs = (double)S.fs;
  if (threadIdx.x == 0) {
    long long oldest = (long long)(st->synthesized_sample / (fp * fs)) - 1;
    if (oldest < 0) oldest = 0;
    sh_ok = (st->cumulative_frame + n - oldest + 1 > S.cap_frames) ? 0 : 1;
    st->last_add_status = sh_ok;
  }
  __syncthreads();
  if (!sh_ok || n <= 0) return;
  const long long cum_before = st->cumulative_frame;
  // a. frames into the ring
  for (int i = threadIdx.x; i < n; i += blockDim.x) S.f0[(cum_before + 1 + i) % S.cap_frames] = f0[i];
  for (int fr = threadIdx.x / 256; fr < n; fr += blockDim.x / 256) {          // one 256-thread quarter of the CTA per frame row
    const size_t dst = (size_t)((cum_before + 1 + fr) % S.cap_frames) * nb, src = (size_t)fr * nb;
    for (int k = threadIdx.x & 255; k < nb; k += 256) { S.sp[dst + k] = sp[src + k]; S.ap[dst + k] = ap[src + k]; }
  }
  __syncthreads();
  const long long cum = cum_before + n;
  if (cum < 1) {   // first-ever single frame: only the hand-off f0 is recorded
    if (threadIdx.x == 0) { st->cumulative_frame = cum; st->handoff_f0 = f0[n - 1]; st->handoff = 1; }
    return;
  }
  if (threadIdx.x == 0) {
    long long first_frame = cum - n;
    long long start = (long long)ceil((double)first_frame * fp * fs);
    if (start < 0) start = 0;
    long long end = (long long)ceil((double)cum * fp * fs);
    sh_first_frame = first_frame; sh_start = start; sh_ns = (int)(end - start); sh_hf = st->handoff;
    sh_handoff_f0 = st->handoff_f0;
  }
  __syncthreads();
  const int ns = sh_ns, hf = sh_hf;
  const long long start = sh_start;
  const long long cum0 = sh_first_frame < 0 ? 0 : sh_first_frame;
  const int nc = n + hf;
  const double hf0 = sh_handoff_f0;
  // c. sample-rate f0 / vuv (coarse axis evaluated on the fly)
  // every product below is rounded on its own (__dmul_rn): nvcc would otherwise fuse `t - m * fp` into one FMA and the
  // exact-midpoint voiced/unvoiced tie (s == 0.5) would resolve differently from the CPU code
  auto ct = [&](int j) { return j == 0 ? __dmul_rn((double)cum0, fp) : __dmul_rn((double)(j - hf + cum0 + hf), fp); };
  auto cf = [&](int j) { return (hf && j == 0) ? hf0 : f0[j - hf]; };
  for (int i = threadIdx.x; i < ns; i += blockDim.x) {
    double t = (double)(i + start) / fs;
    int lo = 0, hi = nc;
    while (lo < hi) { int mid = (lo + hi) >> 1; if (ct(mid) <= t) lo = mid + 1; else hi = mid; }
    int k = lo < 1 ? 1 : (lo > nc - 1 ? nc - 1 : lo);
    double x0 = ct(k - 1), x1 = ct(k);
    double s = __ddiv_rn(__dsub_rn(t, x0), __dsub_rn(x1, x0));
    double fa = cf(k - 1), fb = cf(k);
    double va = fa == 0.0 ? 0.0 : 1.0, vb = fb == 0.0 ? 0.0 : 1.0;
    double fi = __dadd_rn(fa, __dmul_rn(s, __dsub_rn(fb, fa)));      // no FMA contraction: must round like the CPU code
    double vi = __dadd_rn(va, __dmul_rn(s, __dsub_rn(vb, va)));
    vi = vi > 0.5 ? 1.0 : 0.0;
    S.if0[i] = vi == 0.0 ? kDefaultF0 : fi;
    S.ivuv[i] = vi;
  }
  __syncthreads();
  // d. total phase = hand-off phase + prefix sum of the increments in a FIXED blocked order (256-sample blocks
  //    left to right, then block totals left to right): bit-identical to the oracle, which matters because the
  //    unvoiced default f0 puts every pulse exactly on a 2*pi multiple (DESIGN.md, "discrete decisions").
  const int np_ = ns + hf;
  {
    const int BLK = 256;
    const int nblk = (np_ + BLK - 1) / BLK;
    double* totals = scan_scratch;                       // nblk <= 1024 (max_samples_per_add / 256)
    // increments first, by all threads (the FP64 division is the long-latency part); the per-block running sums below are then a
    // plain load-add-store chain.  Same values, same order of additions as before (and as the oracle).
    for (int i = threadIdx.x; i < np_; i += blockDim.x) S.tp[i] = i == 0 ? 0.0 : 2.0 * kPi * S.if0[i - hf] / fs;
    __syncthreads();
    for (int b = threadIdx.x; b < nblk; b += blockDim.x) {
      int b0 = b * BLK, b1 = min(b0 + BLK, np_);
      double local = 0.0;
      int i = b0;
      for (; i + 8 <= b1; i += 8) {
        double v[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) v[j] = S.tp[i + j];
#pragma unroll
        for (int j = 0; j < 8; ++j) { local = __dadd_rn(local, v[j]); S.tp[i + j] = local; }
      }
      for (; i < b1; ++i) { local = __dadd_rn(local, S.tp[i]); S.tp[i] = local; }
      totals[b] = local;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
      double base = hf == 1 ? st->handoff_phase : 2.0 * kPi * S.if0[0] / fs;
      for (int b = 0; b < nblk; ++b) { double t = totals[b]; totals[b] = base; base = __dadd_rn(base, t); }
    }
    __syncthreads();
    for (int i = threadIdx.x; i < np_; i += blockDim.x) S.tp[i] = __dadd_rn(totals[i / BLK], S.tp[i]);
    __syncthreads();
  }
  // e. ordered pulse compaction
  int per = (np_ - 1 + blockDim.x - 1) / blockDim.x;
  int lo = threadIdx.x * per, hi = min(lo + per, np_ - 1);
  int cnt = 0;
  for (int i = lo; i < hi; ++i) {
    double a = fmod(S.tp[i], 2.0 * kPi), b = fmod(S.tp[i + 1], 2.0 * kPi);
    cnt += fabs(b - a) > kPi ? 1 : 0;
  }
  int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  int inc = cnt;
  for (int o = 1; o < 32; o <<= 1) { int v = __shfl_up_sync(0xffffffffu, inc, o); if (lane >= o) inc += v; }
  if (lane == 31) wsum[w] = inc;
  __syncthreads();
  if (w == 0) {
    int v = wsum[lane], iv = v;
    for (int o = 1; o < 32; o <<= 1) { int u = __shfl_up_sync(0xffffffffu, iv, o); if (lane >= o) iv += u; }
    wsum[lane] = iv - v;
    if (lane == 31) sh_total = iv;
  }
  __syncthreads();
  const long long base_pulse = st->n_pulses;
  int pos = wsum[w] + inc - cnt;
  for (int i = lo; i < hi; ++i) {
    double a = fmod(S.tp[i], 2.0 * kPi), b = fmod(S.tp[i + 1], 2.0 * kPi);
    if (fabs(b - a) > kPi) {
      double t = (double)(i + start) / fs - (double)hf / fs;
      long long idx = matlab_round(t * fs);
      long long li = idx - start;
      if (li < 0) li = 0;
      if (li >= ns) li = ns - 1;
      int slot = (int)((base_pulse + pos) % S.cap_pulses);
      S.p_time[slot] = t; S.p_index[slot] = idx; S.p_vuv[slot] = S.ivuv[li] > 0.5 ? 1 : 0;
      ++pos;
    }
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    int total = sh_total;
    if (total > 0) st->last_location = S.p_index[(base_pulse + total - 1) % S.cap_pulses];
    st->n_pulses = base_pulse + total;
    st->handoff_phase = S.tp[np_ - 1];
    st->handoff_f0 = f0[n - 1];
    st->handoff = 1;
    st->cumulative_frame = cum;
  }
}

// ------------------------------------------------------------------------------------ noise stream
__device__ inline void xs_step(uint32_t& x, uint32_t& y, uint32_t& z, uint32_t& w) {
  uint32_t t = x ^ (x << 11);
  x = y; y = z; z = w;
  w = (w ^ (w >> 19)) ^ (t ^ (t >> 8));
}

// state <- M * state over GF(2); M: 128 rows x 4 words, row r = output bit r (word r/32, bit r%32)
__device__ inline void gf2_apply(const uint32_t* __restrict__ M, uint32_t s[4]) {
  uint32_t o[4] = {0, 0, 0, 0};
  for (int r = 0; r < 128; ++r) {
    const uint32_t* row = M + r * 4;
    uint32_t v = (row[0] & s[0]) ^ (row[1] & s[1]) ^ (row[2] & s[2]) ^ (row[3] & s[3]);
    o[r >> 5] |= (uint32_t)(__popc(v) & 1) << (r & 31);
  }
  s[0] = o[0]; s[1] = o[1]; s[2] = o[2]; s[3] = o[3];
}

// Bulk generation of `gridDim.x` tiles of kNoiseTile stream positions starting at base_pos, all tiles in parallel:
// CTA b jumps the base state ahead by b tiles (tile-stride matrices), thread t by another 32 t positions.
// state_in/state_out are separate slots so that the read of the base state never races the write of the next one.
__global__ void __launch_bounds__(256) k_synth_noise(SynthDev S, const uint32_t* __restrict__ jump /*[8][128][4]: T^(384 * 2^j)*/,
                                                    const uint32_t* __restrict__ jump_tile /*[16][128][4]: T^(12 * 8192 * 2^j)*/,
                                                    long long base_pos, int slot_in) {
  SynthState* st = S.state;
  uint32_t s[4] = {st->rng_state[slot_in][0], st->rng_state[slot_in][1], st->rng_state[slot_in][2], st->rng_state[slot_in][3]};
  const int tile = blockIdx.x;
  for (int j = 0; j < 16; ++j) if (tile & (1 << j)) gf2_apply(jump_tile + j * 512, s);
  for (int j = 0; j < 8; ++j) if (threadIdx.x & (1 << j)) gf2_apply(jump + j * 512, s);
  long long pos0 = base_pos + (long long)tile * kNoiseTile + (long long)threadIdx.x * 32;
  for (int i = 0; i < 32; ++i) {
    uint32_t tmp = 0;
#pragma unroll
    for (int k = 0; k < 12; ++k) { xs_step(s[0], s[1], s[2], s[3]); tmp += s[3] >> 4; }
    S.noise[(pos0 + i) % S.cap_noise] = tmp;
  }
  if (tile == (int)gridDim.x - 1 && threadIdx.x == 255) {
    st->rng_state[slot_in ^ 1][0] = s[0]; st->rng_state[slot_in ^ 1][1] = s[1];
    st->rng_state[slot_in ^ 1][2] = s[2]; st->rng_state[slot_in ^ 1][3] = s[3];
  }
}

// ------------------------------------------------------------------------------------ plan
__global__ void k_synth_plan(SynthDev S, int max_blocks) {
  if (threadIdx.x != 0) return;
  SynthState* st = S.state;
  const int B = S.buffer_size;
  long long s0 = st->synthesized_sample;
  long long nblocks = 0;
  if (st->n_pulses > 0 && st->last_location - s0 - 1 >= 0) nblocks = (st->last_location - s0 - 1) / B;
  if (nblocks > max_blocks) nblocks = max_blocks;
  long long first = st->next_pulse, count = 0;
  while (true) {
    long long limit = s0 + nblocks * B;
    // pulses [first, first+count) with index < limit (indices ascending)
    long long lo = first, hi = st->n_pulses;
    while (lo < hi) { long long mid = (lo + hi) >> 1; if (S.p_index[mid % S.cap_pulses] < limit) lo = mid + 1; else hi = mid; }
    count = lo - first;
    if (count <= S.max_pulses || nblocks == 0) break;
    --nblocks;
  }
  if (nblocks == 0) count = 0;
  st->plan_blocks = (int)nblocks;
  st->plan_first = first;
  st->plan_count = (int)count;
}

// ------------------------------------------------------------------------------------ per-pulse response
constexpr int kPulseGrid = 264;      // 2 CTAs x 132 SMs; more pulses than that in one drain are handled by the grid-stride loop
__global__ void __launch_bounds__(256) k_synth_pulse(SynthDev S, const double2* __restrict__ tw) {
  extern __shared__ double2 sm2[];
  SynthState* st = S.state;
  const int plan_count = st->plan_count;
  const int n = S.fft_size, nb = n / 2 + 1, lg = ilog2(n);
  double2* A = sm2;
  double2* Nz = sm2 + n;
  double* spec = (double*)(sm2 + 2 * n);
  double* apr = spec + nb + 1;
  double* periodic = apr + nb + 1;
  double* scratch = periodic + n;
  // grid-stride over the planned pulses: the grid is sized for a typical chunk (one wave of CTAs), not for the worst case --
  // 2048 mostly-empty CTAs of 50 KB shared memory each used to queue behind the stage-2 conv CTAs just to exit
  for (int pq = blockIdx.x; pq < plan_count; pq += gridDim.x) {
  __syncthreads();
  const long long p = st->plan_first + pq;
  const int slot = (int)(p % S.cap_pulses);
  const double t = S.p_time[slot];
  const int vuv = S.p_vuv[slot];
  const long long idx = S.p_index[slot];
  long long nxt = S.p_index[(p + 1) % S.cap_pulses];
  int noise_size = (int)(nxt - idx);
  if (noise_size < 1) noise_size = 1;
  if (noise_size > n) noise_size = n;
  const long long qpos = idx < 0 ? 0 : idx;
  long long fl = (long long)(t / S.frame_period);
  long long ce = (long long)ceil(t / S.frame_period);
  const double interp = t / S.frame_period - fl;
  const long long cum = st->cumulative_frame;
  if (fl > cum) fl = cum;
  if (ce > cum) ce = cum;
  const float* sp0 = S.sp + (size_t)(fl % S.cap_frames) * nb; const float* sp1 = S.sp + (size_t)(ce % S.cap_frames) * nb;
  const float* ap0 = S.ap + (size_t)(fl % S.cap_frames) * nb; const float* ap1 = S.ap + (size_t)(ce % S.cap_frames) * nb;
  for (int i = threadIdx.x; i < nb; i += blockDim.x) {
    double sv, av;
    if (fl == ce) { sv = fabs((double)sp0[i]); av = safe_ap((double)ap0[i]); }
    else {
      sv = (1.0 - interp) * fabs((double)sp0[i]) + interp * fabs((double)sp1[i]);
      av = (1.0 - interp) * safe_ap((double)ap0[i]) + interp * safe_ap((double)ap1[i]);
    }
    spec[i] = sv; apr[i] = av * av;
  }
  __syncthreads();
  // periodic response
  const bool has_periodic = !(vuv == 0 || apr[0] > 0.999);
  if (!has_periodic) {
    for (int i = threadIdx.x; i < n; i += blockDim.x) periodic[i] = 0.0;
  } else {
    for (int i = threadIdx.x; i < nb; i += blockDim.x) A[i] = make_double2(log(spec[i] * (1.0 - apr[i]) + kSafeMin) / 2.0, 0.0);
    min_phase_smem(A, n, lg, tw);
    irfft_smem(A, n, lg, tw);
    double part = 0.0;
    for (int i = n / 2 + threadIdx.x; i < n; i += blockDim.x) part += A[i - n / 2].x;      // periodic[i] = tmp[i - n/2]
    double dc = block_sum(part, scratch);
    for (int i = threadIdx.x; i < n; i += blockDim.x)
      periodic[i] = i < n / 2 ? 0.0 : A[i - n / 2].x - dc * S.dc_remover[i - n / 2];
  }
  __syncthreads();
  // aperiodic response: zero-mean noise of length noise_size
  double part = 0.0;
  for (int i = threadIdx.x; i < noise_size; i += blockDim.x)
    part += (double)S.noise[(qpos + i) % S.cap_noise] / 268435456.0 - 6.0;
  double avg = block_sum(part, scratch) / noise_size;
  for (int i = threadIdx.x; i < n; i += blockDim.x) {
    double v = 0.0;
    if (i < noise_size) v = ((double)S.noise[(qpos + i) % S.cap_noise] / 268435456.0 - 6.0) - avg;
    Nz[i] = make_double2(v, 0.0);
  }
  fft_smem(Nz, n, lg, -1, tw);
  for (int i = threadIdx.x; i < nb; i += blockDim.x) {
    double v = vuv != 0 ? log(spec[i] * apr[i]) / 2.0 : log(spec[i]) / 2.0;
    A[i] = make_double2(v, 0.0);
  }
  min_phase_smem(A, n, lg, tw);
  for (int i = threadIdx.x; i < nb; i += blockDim.x) {
    double2 m = A[i], z = Nz[i];
    A[i] = make_double2(m.x * z.x - m.y * z.y, m.x * z.y + m.y * z.x);
  }
  irfft_smem(A, n, lg, tw);
  const double sq = sqrt((double)noise_size);
  double* resp = S.resp + (size_t)pq * n;
  for (int i = threadIdx.x; i < n; i += blockDim.x) {
    double aper = i < n / 2 ? A[i + n / 2].x : A[i - n / 2].x;
    resp[i] = (periodic[i] * sq + aper) / n;
  }
  }
}

// ------------------------------------------------------------------------------------ overlap-add
// absolute sample a = s0 + j for j in [0, nblocks*B + carry_len): carry_in + pulses (in pulse order).
__global__ void __launch_bounds__(256) k_synth_ola(SynthDev S, double* __restrict__ out, int out_cap_samples, int phase) {
  SynthState* st = S.state;
  const int B = S.buffer_size, n = S.fft_size;
  const int nblocks = st->plan_blocks, count = st->plan_count;
  const long long s0 = st->synthesized_sample;
  const long long first = st->plan_first;
  const int total = nblocks * B + S.carry_len;
  const double* cin = S.carry[st->carry_sel];
  double* cout = S.carry[st->carry_sel ^ 1];
  if (phase == 0) {
    if (nblocks == 0) return;
    for (int j = blockIdx.x * blockDim.x + threadIdx.x; j < total; j += gridDim.x * blockDim.x) {
      long long a = s0 + j;
      double v = j < S.carry_len ? cin[j] : 0.0;
      // pulses with idx in [a - n/2, a + n/2 - 1]
      long long lo = 0, hi = count;
      long long want = a - n / 2;
      while (lo < hi) { long long mid = (lo + hi) >> 1; if (S.p_index[(first + mid) % S.cap_pulses] < want) lo = mid + 1; else hi = mid; }
      for (long long q = lo; q < count; ++q) {
        long long idx = S.p_index[(first + q) % S.cap_pulses];
        if (idx > a + n / 2 - 1) break;
        long long blockstart = idx < s0 ? s0 : s0 + ((idx - s0) / B) * B;
        if (a < blockstart) continue;
        long long off = idx - n / 2 + 1;     // absolute sample of response[0]
        v += S.resp[(size_t)q * n + (a - off)];
      }
      if (j < nblocks * B) { if (j < out_cap_samples) out[j] = v; }
      else cout[j - nblocks * B] = v;
    }
  } else {
    if (blockIdx.x == 0 && threadIdx.x == 0 && nblocks > 0) {
      st->synthesized_sample = s0 + (long long)nblocks * B;
      st->next_pulse = first + count;
      st->carry_sel ^= 1;
    }
    if (blockIdx.x == 0 && threadIdx.x == 0) st->blocks_out = nblocks;
  }
}

// ------------------------------------------------------------------------------------ host side
static void gf2_mul(const uint32_t* A, const uint32_t* Bm, uint32_t* C) {   // C = A * B (apply B first), 128x128 bit rows
  // column extraction of B is awkward; use C row r = XOR over set bits k of A row r of B row k
  for (int r = 0; r < 128; ++r) {
    uint32_t acc[4] = {0, 0, 0, 0};
    for (int k = 0; k < 128; ++k)
      if (A[r * 4 + (k >> 5)] >> (k & 31) & 1) for (int w = 0; w < 4; ++w) acc[w] ^= Bm[k * 4 + w];
    for (int w = 0; w < 4; ++w) C[r * 4 + w] = acc[w];
  }
}

// jump[j] = T^(12*32*2^j), T = one xorshift128 step on the 128-bit state (x,y,z,w) = words 0..3
static void build_jump_matrices(std::vector<uint32_t>& jump) {
  std::vector<uint32_t> T(512, 0), P(512), Q(512);
  // build T column by column: apply one step to each basis state
  for (int c = 0; c < 128; ++c) {
    uint32_t s[4] = {0, 0, 0, 0};
    s[c >> 5] = 1u << (c & 31);
    uint32_t t = s[0] ^ (s[0] << 11);
    uint32_t nx = s[1], ny = s[2], nz = s[3];
    uint32_t nw = (s[3] ^ (s[3] >> 19)) ^ (t ^ (t >> 8));
    uint32_t o[4] = {nx, ny, nz, nw};
    for (int r = 0; r < 128; ++r) if (o[r >> 5] >> (r & 31) & 1) T[r * 4 + (c >> 5)] |= 1u << (c & 31);
  }
  // P = T^384 by square-and-multiply (384 = 256 + 128)
  std::vector<uint32_t> pw = T;          // T^(2^k)
  std::vector<uint32_t> acc; bool have = false;
  for (int bit = 0; bit < 9; ++bit) {
    if ((384 >> bit) & 1) {
      if (!have) { acc = pw; have = true; } else { gf2_mul(pw.data(), acc.data(), Q.data()); acc = Q; }
    }
    gf2_mul(pw.data(), pw.data(), Q.data()); pw = Q;
  }
  // jump[0..8): T^(384 * 2^j) (32 positions * 2^j);  jump[8..24): T^(12 * 8192 * 2^j) = (T^384)^(256 * 2^j)
  jump.resize(24 * 512);
  P = acc;
  for (int j = 0; j < 24; ++j) {
    memcpy(&jump[j * 512], P.data(), 512 * sizeof(uint32_t));
    gf2_mul(P.data(), P.data(), Q.data()); P = Q;
  }
}

int synth_module_init(Engine* e) {
  if (e->d_jump) return 0;
  std::vector<uint32_t> jump;
  build_jump_matrices(jump);
  RYK_CUDA(cudaMalloc(&e->d_jump, jump.size() * sizeof(uint32_t)));
  RYK_CUDA(cudaMemcpy(e->d_jump, jump.data(), jump.size() * sizeof(uint32_t), cudaMemcpyHostToDevice));
  RYK_CUDA(cudaFuncSetAttribute(k_synth_pulse, cudaFuncAttributeMaxDynamicSharedMemorySize, 160 * 1024));
  return 0;
}

static size_t pulse_smem_bytes(int n) {
  int nb = n / 2 + 1;
  return sizeof(double2) * 2 * n + sizeof(double) * (2 * (nb + 1) + n + 64);
}

int synth_create(Engine* e, int fs, double frame_period_ms, int fft_size, int buffer_size, int ring_frames, Synth** out) {
  if (synth_module_init(e)) return -1;
  RYK_CHECK(fft_size >= 64 && fft_size <= kTwiddleN && (fft_size & (fft_size - 1)) == 0, "unsupported synthesis fft size");
  Synth* s = new Synth();
  SynthDev& D = s->dev;
  D.fs = fs; D.fft_size = fft_size; D.buffer_size = buffer_size; D.frame_period = frame_period_ms / 1000.0;
  D.cap_frames = ring_frames; D.cap_pulses = 1 << 15; D.cap_noise = 1 << 22; D.max_pulses = 2048;
  D.carry_len = buffer_size + fft_size;
  D.max_samples_per_add = 1 << 17;
  int nb = fft_size / 2 + 1;
  auto A = [&](void** p, size_t bytes) -> int { RYK_CUDA(cudaMalloc(p, bytes)); RYK_CUDA(cudaMemset(*p, 0, bytes)); s->allocs.push_back(*p); return 0; };
  if (A((void**)&D.state, sizeof(SynthState))) return -1;
  if (A((void**)&D.f0, sizeof(double) * ring_frames)) return -1;
  if (A((void**)&D.sp, sizeof(float) * (size_t)ring_frames * nb)) return -1;
  if (A((void**)&D.ap, sizeof(float) * (size_t)ring_frames * nb)) return -1;
  if (A((void**)&D.p_index, sizeof(long long) * D.cap_pulses)) return -1;
  if (A((void**)&D.p_time, sizeof(double) * D.cap_pulses)) return -1;
  if (A((void**)&D.p_vuv, sizeof(int) * D.cap_pulses)) return -1;
  if (A((void**)&D.noise, sizeof(uint32_t) * D.cap_noise)) return -1;
  if (A((void**)&D.if0, sizeof(double) * D.max_samples_per_add)) return -1;
  if (A((void**)&D.ivuv, sizeof(double) * D.max_samples_per_add)) return -1;
  if (A((void**)&D.tp, sizeof(double) * (D.max_samples_per_add + 2))) return -1;
  if (A((void**)&D.resp, sizeof(double) * (size_t)D.max_pulses * fft_size)) return -1;
  if (A((void**)&D.carry[0], sizeof(double) * D.carry_len)) return -1;
  if (A((void**)&D.carry[1], sizeof(double) * D.carry_len)) return -1;
  if (A((void**)&D.dc_remover, sizeof(double) * (fft_size / 2))) return -1;
  std::vector<double> dc(fft_size / 2);
  double sum = 0.0;
  for (int i = 0; i < fft_size / 2; ++i) { dc[i] = 0.5 - 0.5 * cos(2.0 * kPi * (i + 1.0) / (1.0 + fft_size / 2)); sum += dc[i]; }
  for (auto& v : dc) v /= sum;
  RYK_CUDA(cudaMemcpy(D.dc_remover, dc.data(), sizeof(double) * dc.size(), cudaMemcpyHostToDevice));
  SynthState init;
  memset(&init, 0, sizeof(init));
  init.cumulative_frame = -1;
  init.rng_state[0][0] = 123456789u; init.rng_state[0][1] = 362436069u; init.rng_state[0][2] = 521288629u; init.rng_state[0][3] = 88675123u;
  RYK_CUDA(cudaMemcpy(D.state, &init, sizeof(init), cudaMemcpyHostToDevice));
  s->host_cum_frames = -1; s->host_noise_generated = 0; s->host_noise_slot = 0;
  *out = s;
  return 0;
}

void synth_destroy(Synth* s) {
  if (!s) return;
  for (void* p : s->allocs) cudaFree(p);
  delete s;
}

// Stream-ordered: append n frames (device pointers). Also tops up the noise ring to the new end sample.
// Host-side bookkeeping of an AddParameters call (frame counter) + the rare bulk noise top-up; never captured in a graph.
int synth_host_advance(Engine* e, Synth* s, int n, cudaStream_t st) {
  SynthDev& D = s->dev;
  RYK_CHECK((long long)n * D.frame_period * D.fs + 2 < D.max_samples_per_add, "too many frames in one AddParameters call");
  static_assert((1 << 17) / 256 <= 1024, "block totals must fit the scan scratch");
  s->host_cum_frames += n;
  long long need = (long long)ceil((double)(s->host_cum_frames < 0 ? 0 : s->host_cum_frames) * D.frame_period * D.fs) + D.fft_size + 2;
  if (need > s->host_noise_generated) {
    // top the ring up in one bulk launch: half a ring ahead (cap_noise / 2 positions = 87 s of audio at 24 kHz),
    // so the noise stream costs one ~1 ms launch every few hundred chunks instead of a kernel per chunk
    int tiles = D.cap_noise / 2 / kNoiseTile;
    k_synth_noise<<<tiles, 256, 0, st>>>(D, e->d_jump, e->d_jump + 8 * 512, s->host_noise_generated, s->host_noise_slot);
    s->host_noise_generated += (long long)tiles * kNoiseTile;
    s->host_noise_slot ^= 1;
    e->launches++;
    RYK_CUDA(cudaGetLastError());
  }
  return 0;
}

// The device side of AddParameters (graph-capturable: fixed arguments, no host state).
int synth_add_kernel(Engine* e, Synth* s, const double* d_f0, int n, const float* d_sp, const float* d_ap, cudaStream_t st) {
  k_synth_add<<<1, 1024, 0, st>>>(s->dev, d_f0, n, d_sp, d_ap);
  RYK_CUDA(cudaGetLastError());
  return 0;
}

// Stream-ordered: append n frames (device pointers). Also tops up the noise ring to the new end sample.
int synth_add_async(Engine* e, Synth* s, const double* d_f0, int n, const float* d_sp, const float* d_ap, cudaStream_t st) {
  if (synth_host_advance(e, s, n, st)) return -1;
  return synth_add_kernel(e, s, d_f0, n, d_sp, d_ap, st);
}

// Stream-ordered: emit up to max_blocks blocks into d_out (doubles); the count lands in state->blocks_out.
int synth_drain_async(Engine* e, Synth* s, double* d_out, int max_blocks, cudaStream_t st) {
  SynthDev& D = s->dev;
  k_synth_plan<<<1, 32, 0, st>>>(D, max_blocks);
  k_synth_pulse<<<D.max_pulses < kPulseGrid ? D.max_pulses : kPulseGrid, 256, pulse_smem_bytes(D.fft_size), st>>>(D, e->d_twiddle);
  int total = max_blocks * D.buffer_size + D.carry_len;
  k_synth_ola<<<(total + 255) / 256, 256, 0, st>>>(D, d_out, max_blocks * D.buffer_size, 0);
  k_synth_ola<<<1, 32, 0, st>>>(D, d_out, 0, 1);
  RYK_CUDA(cudaGetLastError());
  return 0;
}


// ------------------------------------------------------------------------------------ offline Synthesis()
// SURVEY 8(f) rank 3: Vocoder.decode = pyworld.synthesize (realtime_voice_conversion/yukarin_wrapper/vocoder.py:50-62),
// WORLD synthesis.cpp Synthesis(): whole-utterance time base (with the extrapolated coarse point and the lowest-f0 clamp),
// fractional pulse time shift, Hanning dc-remover over the whole fft_size, plain overlap-add.  Shares the per-pulse
// machinery (shared-memory FP64 FFT chains, position-addressed xorshift128 noise) with the realtime synthesizer above.
struct OfflineDev {
  int fs, fft_size, n_frames, y_length;
  double frame_period;                                   // seconds
  const double* f0; const float* sp; const float* ap;    // [n_frames], [n_frames][nb]
  double *if0, *ivuv, *tp, *totals;                      // [y_length] x 3, [ceil(y_length / 256)]
  long long* p_index; double* p_shift; int* p_vuv; int* n_pulses;
  const uint32_t* noise; int cap_noise;
  const double* dc_remover;                              // [fft_size]
  double* resp;                                          // [batch][fft_size]
  double* y;
};

__global__ void __launch_bounds__(1024) k_off_timebase(OfflineDev S) {
  __shared__ int wsum[32];
  __shared__ int sh_total;
  const int nf = S.n_frames, ny = S.y_length;
  const double fp = S.frame_period, fs = (double)S.fs;
  const double lowest_f0 = fs / S.fft_size + 1.0;
  const int nc = nf + 1;
  auto cfr = [&](int j) { double v = S.f0[j]; return v < lowest_f0 ? 0.0 : v; };
  auto cf = [&](int j) { return j < nf ? cfr(j) : (nf >= 2 ? __dsub_rn(__dmul_rn(cfr(nf - 1), 2.0), cfr(nf - 2)) : cfr(0)); };
  auto cvr = [&](int j) { return cfr(j) == 0.0 ? 0.0 : 1.0; };
  auto cv = [&](int j) { return j < nf ? cvr(j) : (nf >= 2 ? cvr(nf - 1) * 2.0 - cvr(nf - 2) : cvr(0)); };
  auto ct = [&](int j) { return __dmul_rn((double)j, fp); };
  for (int i = threadIdx.x; i < ny; i += blockDim.x) {
    const double t = (double)i / fs;
    int lo = 0, hi = nc;
    while (lo < hi) { int mid = (lo + hi) >> 1; if (ct(mid) <= t) lo = mid + 1; else hi = mid; }
    const int k = lo < 1 ? 1 : (lo > nc - 1 ? nc - 1 : lo);
    const double x0 = ct(k - 1), x1 = ct(k);
    const double sx = __ddiv_rn(__dsub_rn(t, x0), __dsub_rn(x1, x0));
    const double fa = cf(k - 1), fb = cf(k), va = cv(k - 1), vb = cv(k);
    const double fi = __dadd_rn(fa, __dmul_rn(sx, __dsub_rn(fb, fa)));       // no FMA contraction (see k_synth_add)
    double vi = __dadd_rn(va, __dmul_rn(sx, __dsub_rn(vb, va)));
    vi = vi > 0.5 ? 1.0 : 0.0;
    S.if0[i] = vi == 0.0 ? kDefaultF0 : fi;
    S.ivuv[i] = vi;
  }
  __syncthreads();
  // total phase: inclusive prefix sum of 2 pi f0 / fs in the fixed blocked order (256-sample blocks, then block totals)
  const int BLK = 256, nblk = (ny + BLK - 1) / BLK;
  for (int b = threadIdx.x; b < nblk; b += blockDim.x) {
    const int b0 = b * BLK, b1 = min(b0 + BLK, ny);
    double local = 0.0;
    for (int i = b0; i < b1; ++i) { local = __dadd_rn(local, 2.0 * kPi * S.if0[i] / fs); S.tp[i] = local; }
    S.totals[b] = local;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    double base = 0.0;
    for (int b = 0; b < nblk; ++b) { const double t = S.totals[b]; S.totals[b] = base; base = __dadd_rn(base, t); }
  }
  __syncthreads();
  for (int i = threadIdx.x; i < ny; i += blockDim.x) S.tp[i] = __dadd_rn(S.totals[i / BLK], S.tp[i]);
  __syncthreads();
  // ordered pulse compaction
  const int per = (ny - 1 + blockDim.x - 1) / blockDim.x;
  const int lo = threadIdx.x * per, hi = min(lo + per, ny - 1);
  int cnt = 0;
  for (int i = lo; i < hi; ++i) {
    const double a = fmod(S.tp[i], 2.0 * kPi), b = fmod(S.tp[i + 1], 2.0 * kPi);
    cnt += fabs(b - a) > kPi ? 1 : 0;
  }
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  int inc = cnt;
  for (int o = 1; o < 32; o <<= 1) { int v = __shfl_up_sync(0xffffffffu, inc, o); if (lane >= o) inc += v; }
  if (lane == 31) wsum[w] = inc;
  __syncthreads();
  if (w == 0) {
    int v = wsum[lane], iv = v;
    for (int o = 1; o < 32; o <<= 1) { int u = __shfl_up_sync(0xffffffffu, iv, o); if (lane >= o) iv += u; }
    wsum[lane] = iv - v;
    if (lane == 31) sh_total = iv;
  }
  __syncthreads();
  int pos = wsum[w] + inc - cnt;
  for (int i = lo; i < hi; ++i) {
    const double a = fmod(S.tp[i], 2.0 * kPi), b = fmod(S.tp[i + 1], 2.0 * kPi);
    if (fabs(b - a) > kPi) {
      const double y1 = a - 2.0 * kPi, y2 = b;
      const double x = -y1 / (y2 - y1);
      S.p_index[pos] = i; S.p_shift[pos] = x / fs; S.p_vuv[pos] = S.ivuv[i] > 0.5 ? 1 : 0;
      ++pos;
    }
  }
  if (threadIdx.x == 0) *S.n_pulses = sh_total;
}

// one CTA per pulse of the batch [first, first + count)
__global__ void __launch_bounds__(256) k_off_pulse(OfflineDev S, int first, int count, const double2* __restrict__ tw) {
  extern __shared__ double2 sm2[];
  if ((int)blockIdx.x >= count) return;
  const int n = S.fft_size, nb = n / 2 + 1, lg = ilog2(n);
  double2* A = sm2;
  double2* Nz = sm2 + n;
  double* spec = (double*)(sm2 + 2 * n);
  double* apr = spec + nb + 1;
  double* periodic = apr + nb + 1;
  double* scratch = periodic + n;
  const int np_ = *S.n_pulses;
  const int p = first + blockIdx.x;
  const long long idx = S.p_index[p];
  const long long nxt = S.p_index[p + 1 < np_ ? p + 1 : np_ - 1];
  int noise_size = (int)(nxt - idx);
  if (noise_size > n) noise_size = n;
  const int vuv = S.p_vuv[p];
  const double t = (double)idx / (double)S.fs;
  int fl = (int)floor(t / S.frame_period), ce = (int)ceil(t / S.frame_period);
  if (fl > S.n_frames - 1) fl = S.n_frames - 1;
  if (ce > S.n_frames - 1) ce = S.n_frames - 1;
  const double interp = t / S.frame_period - fl;
  const float* sp0 = S.sp + (size_t)fl * nb; const float* sp1 = S.sp + (size_t)ce * nb;
  const float* ap0 = S.ap + (size_t)fl * nb; const float* ap1 = S.ap + (size_t)ce * nb;
  for (int i = threadIdx.x; i < nb; i += blockDim.x) {
    double sv, av;
    if (fl == ce) { sv = fabs((double)sp0[i]); av = safe_ap((double)ap0[i]); }
    else {
      sv = (1.0 - interp) * fabs((double)sp0[i]) + interp * fabs((double)sp1[i]);
      av = (1.0 - interp) * safe_ap((double)ap0[i]) + interp * safe_ap((double)ap1[i]);
    }
    spec[i] = sv; apr[i] = av * av;
  }
  __syncthreads();
  const bool has_periodic = !(vuv == 0 || apr[0] > 0.999);
  if (!has_periodic) {
    for (int i = threadIdx.x; i < n; i += blockDim.x) periodic[i] = 0.0;
  } else {
    for (int i = threadIdx.x; i < nb; i += blockDim.x) A[i] = make_double2(log(spec[i] * (1.0 - apr[i]) + kSafeMin) / 2.0, 0.0);
    min_phase_smem(A, n, lg, tw);
    const double coef = 2.0 * kPi * S.p_shift[p] * S.fs / n;          // linear-phase fractional delay
    for (int i = threadIdx.x; i < nb; i += blockDim.x) {
      const double2 v = A[i];
      const double re2 = cos(coef * i), im2 = sqrt(1.0 - re2 * re2);
      A[i] = make_double2(v.x * re2 + v.y * im2, v.y * re2 - v.x * im2);
    }
    irfft_smem(A, n, lg, tw);
    double part = 0.0;
    for (int i = n / 2 + threadIdx.x; i < n; i += blockDim.x) part += A[i - n / 2].x;      // fftshift: periodic[i] = tmp[i - n/2]
    const double dc = block_sum(part, scratch);
    for (int i = threadIdx.x; i < n; i += blockDim.x)
      periodic[i] = i < n / 2 ? -dc * S.dc_remover[i] : A[i - n / 2].x - dc * S.dc_remover[i];
  }
  __syncthreads();
  double part = 0.0;
  for (int i = threadIdx.x; i < noise_size; i += blockDim.x)
    part += (double)S.noise[(idx + i) % S.cap_noise] / 268435456.0 - 6.0;
  const double avg = noise_size > 0 ? block_sum(part, scratch) / noise_size : block_sum(part, scratch);
  for (int i = threadIdx.x; i < n; i += blockDim.x) {
    double v = 0.0;
    if (i < noise_size) v = ((double)S.noise[(idx + i) % S.cap_noise] / 268435456.0 - 6.0) - avg;
    Nz[i] = make_double2(v, 0.0);
  }
  fft_smem(Nz, n, lg, -1, tw);
  for (int i = threadIdx.x; i < nb; i += blockDim.x) {
    const double v = vuv != 0 ? log(spec[i] * apr[i]) / 2.0 : log(spec[i]) / 2.0;
    A[i] = make_double2(v, 0.0);
  }
  min_phase_smem(A, n, lg, tw);
  for (int i = threadIdx.x; i < nb; i += blockDim.x) {
    const double2 m = A[i], z = Nz[i];
    A[i] = make_double2(m.x * z.x - m.y * z.y, m.x * z.y + m.y * z.x);
  }
  irfft_smem(A, n, lg, tw);
  const double sq = sqrt((double)noise_size);
  double* resp = S.resp + (size_t)blockIdx.x * n;
  for (int i = threadIdx.x; i < n; i += blockDim.x) {
    const double aper = i < n / 2 ? A[i + n / 2].x : A[i - n / 2].x;
    resp[i] = (periodic[i] * sq + aper) / n;
  }
}

// gather overlap-add of one pulse batch, in pulse order (deterministic): y[a] += sum of the batch's responses covering a
__global__ void __launch_bounds__(256) k_off_ola(OfflineDev S, int first, int count) {
  const int n = S.fft_size;
  for (int a = blockIdx.x * blockDim.x + threadIdx.x; a < S.y_length; a += gridDim.x * blockDim.x) {
    // pulses of the batch with idx in [a - n/2, a + n/2 - 1]
    int lo = 0, hi = count;
    const long long want = (long long)a - n / 2;
    while (lo < hi) { int mid = (lo + hi) >> 1; if (S.p_index[first + mid] < want) lo = mid + 1; else hi = mid; }
    double v = S.y[a];
    for (int q = lo; q < count; ++q) {
      const long long idx = S.p_index[first + q];
      if (idx > (long long)a + n / 2 - 1) break;
      v += S.resp[(size_t)q * n + (a - (idx - n / 2 + 1))];
    }
    S.y[a] = v;
  }
}

// Host buffers in, host buffer out (the per-op level of the C ABI).  Returns the number of pulses, < 0 on error.
int world_synthesize_run(Engine* e, const double* f0, int n_frames, const float* sp, const float* ap, int fs, double frame_period_ms,
                         int fft_size, double* y, int y_length, long long* pulse_index, double* pulse_shift, int* pulse_vuv, int max_pulses) {
  if (synth_module_init(e)) return -1;
  { static bool attr_set = false;
    if (!attr_set) { RYK_CUDA(cudaFuncSetAttribute(k_off_pulse, cudaFuncAttributeMaxDynamicSharedMemorySize, 160 * 1024)); attr_set = true; } }
  RYK_CHECK(fft_size >= 64 && fft_size <= kTwiddleN && (fft_size & (fft_size - 1)) == 0, "unsupported synthesis fft size");
  RYK_CHECK(n_frames >= 1 && y_length >= 0 && y_length < (1 << 28), "bad synthesis length");
  if (y_length == 0) return 0;
  cudaStream_t st = e->stream;
  const int n = fft_size, nb = n / 2 + 1;
  if (y_length < 2) { y[0] = 0.0; return 0; }
  std::vector<void*> allocs;
  auto A = [&](void** p, size_t bytes) -> int { RYK_CUDA(cudaMalloc(p, bytes)); allocs.push_back(*p); return 0; };
  auto cleanup = [&]() { for (void* p : allocs) cudaFree(p); };
  OfflineDev S;
  memset(&S, 0, sizeof(S));
  S.fs = fs; S.fft_size = n; S.n_frames = n_frames; S.y_length = y_length; S.frame_period = frame_period_ms / 1000.0;
  const int tiles = (y_length + n + kNoiseTile - 1) / kNoiseTile;
  RYK_CHECK(tiles < 65536, "utterance too long for the noise jump table");
  const int nblk = (y_length + 255) / 256;
  double* d_f0 = nullptr; float *d_sp = nullptr, *d_ap = nullptr; uint32_t* d_noise = nullptr; double* d_dc = nullptr; SynthState* d_state = nullptr;
  int rc = 0;
  const int kBatch = 4096;
  rc |= A((void**)&d_f0, sizeof(double) * n_frames);
  rc |= A((void**)&d_sp, sizeof(float) * (size_t)n_frames * nb);
  rc |= A((void**)&d_ap, sizeof(float) * (size_t)n_frames * nb);
  rc |= A((void**)&S.if0, sizeof(double) * y_length);
  rc |= A((void**)&S.ivuv, sizeof(double) * y_length);
  rc |= A((void**)&S.tp, sizeof(double) * y_length);
  rc |= A((void**)&S.totals, sizeof(double) * nblk);
  rc |= A((void**)&S.p_index, sizeof(long long) * y_length);
  rc |= A((void**)&S.p_shift, sizeof(double) * y_length);
  rc |= A((void**)&S.p_vuv, sizeof(int) * y_length);
  rc |= A((void**)&S.n_pulses, sizeof(int));
  rc |= A((void**)&d_noise, sizeof(uint32_t) * (size_t)tiles * kNoiseTile);
  rc |= A((void**)&d_dc, sizeof(double) * n);
  rc |= A((void**)&d_state, sizeof(SynthState));
  rc |= A((void**)&S.resp, sizeof(double) * (size_t)kBatch * n);
  rc |= A((void**)&S.y, sizeof(double) * y_length);
  if (rc) { cleanup(); return -1; }
  S.f0 = d_f0; S.sp = d_sp; S.ap = d_ap; S.noise = d_noise; S.cap_noise = tiles * kNoiseTile; S.dc_remover = d_dc;
  std::vector<double> dc(n);
  { double sum = 0.0;
    for (int i = 0; i < n / 2; ++i) { dc[i] = 0.5 - 0.5 * cos(2.0 * kPi * (i + 1.0) / (1.0 + n)); dc[n - i - 1] = dc[i]; sum += dc[i] * 2.0; }
    for (int i = 0; i < n / 2; ++i) { dc[i] /= sum; dc[n - i - 1] = dc[i]; } }
  SynthState init;
  memset(&init, 0, sizeof(init));
  init.rng_state[0][0] = 123456789u; init.rng_state[0][1] = 362436069u; init.rng_state[0][2] = 521288629u; init.rng_state[0][3] = 88675123u;
  auto fail = [&](const char* what) { set_error(what); cleanup(); return -1; };
#define OFF_CUDA(x) do { cudaError_t err_ = (x); if (err_ != cudaSuccess) return fail(cudaGetErrorString(err_)); } while (0)
  OFF_CUDA(cudaMemcpyAsync(d_f0, f0, sizeof(double) * n_frames, cudaMemcpyHostToDevice, st));
  OFF_CUDA(cudaMemcpyAsync(d_sp, sp, sizeof(float) * (size_t)n_frames * nb, cudaMemcpyHostToDevice, st));
  OFF_CUDA(cudaMemcpyAsync(d_ap, ap, sizeof(float) * (size_t)n_frames * nb, cudaMemcpyHostToDevice, st));
  OFF_CUDA(cudaMemcpyAsync(d_dc, dc.data(), sizeof(double) * n, cudaMemcpyHostToDevice, st));
  OFF_CUDA(cudaMemcpyAsync(d_state, &init, sizeof(init), cudaMemcpyHostToDevice, st));
  OFF_CUDA(cudaMemsetAsync(S.y, 0, sizeof(double) * y_length, st));
  {
    SynthDev N;
    memset(&N, 0, sizeof(N));
    N.state = d_state; N.noise = d_noise; N.cap_noise = S.cap_noise;
    k_synth_noise<<<tiles, 256, 0, st>>>(N, e->d_jump, e->d_jump + 8 * 512, 0, 0);
  }
  k_off_timebase<<<1, 1024, 0, st>>>(S);
  int np_ = 0;
  OFF_CUDA(cudaMemcpyAsync(&np_, S.n_pulses, sizeof(int), cudaMemcpyDeviceToHost, st));
  OFF_CUDA(cudaStreamSynchronize(st));
  for (int first = 0; first < np_; first += kBatch) {
    const int count = np_ - first < kBatch ? np_ - first : kBatch;
    k_off_pulse<<<count, 256, pulse_smem_bytes(n), st>>>(S, first, count, e->d_twiddle);
    k_off_ola<<<(y_length + 255) / 256, 256, 0, st>>>(S, first, count);
  }
  OFF_CUDA(cudaGetLastError());
  OFF_CUDA(cudaMemcpyAsync(y, S.y, sizeof(double) * y_length, cudaMemcpyDeviceToHost, st));
  const int nq = np_ < max_pulses ? np_ : max_pulses;
  if (pulse_index && nq > 0) OFF_CUDA(cudaMemcpyAsync(pulse_index, S.p_index, sizeof(long long) * nq, cudaMemcpyDeviceToHost, st));
  if (pulse_shift && nq > 0) OFF_CUDA(cudaMemcpyAsync(pulse_shift, S.p_shift, sizeof(double) * nq, cudaMemcpyDeviceToHost, st));
  if (pulse_vuv && nq > 0) OFF_CUDA(cudaMemcpyAsync(pulse_vuv, S.p_vuv, sizeof(int) * nq, cudaMemcpyDeviceToHost, st));
  OFF_CUDA(cudaStreamSynchronize(st));
#undef OFF_CUDA
  cleanup();
  return np_;
}

// ------------------------------------------------------------------------------------ output silence gate
// SURVEY 8(f) rank 2: realtime_voice_conversion/worker/decode_worker.py:53-59 --
//   power = librosa.core.power_to_db(numpy.abs(librosa.stft(wave)) ** 2).mean();  the chunk is dropped if power < -threshold.
// k_ogate_stft : one CTA per STFT frame (n_fft 2048, hop 512, periodic Hann, reflect-centred): FP64 smem FFT -> dB per bin
// k_ogate_mean : top_db clip against the global maximum and the mean; writes {power, pass} -- all on the device, no host sync.
__global__ void __launch_bounds__(256) k_ogate_stft(const double* __restrict__ wave, const int* __restrict__ n_valid, int n, int n_fft, int hop,
                                                   double amin, double* __restrict__ db, double* __restrict__ fmx, const double2* __restrict__ tw) {
  extern __shared__ double2 sm2[];
  __shared__ double red[32];
  if (n_valid && *n_valid < n) return;                 // no chunk was emitted this step
  const int f = blockIdx.x, nb = n_fft / 2 + 1, pad = n_fft / 2, lg = ilog2(n_fft);
  for (int j = threadIdx.x; j < n_fft; j += blockDim.x) {
    int idx = f * hop + j - pad;
    if (idx < 0) idx = -idx;
    if (idx >= n) idx = 2 * (n - 1) - idx;
    if (idx < 0) idx = 0;
    if (idx >= n) idx = n - 1;
    const double w = 0.5 - 0.5 * cos(2.0 * kPi * j / n_fft);
    sm2[j] = make_double2(wave[idx] * w, 0.0);
  }
  fft_smem(sm2, n_fft, lg, -1, tw);
  double mx = -1e300;
  for (int k = threadIdx.x; k < nb; k += blockDim.x) {
    const double2 v = sm2[k];
    const double pw = v.x * v.x + v.y * v.y;
    const double d = 10.0 * log10(pw > amin ? pw : amin);
    db[(size_t)f * nb + k] = d;
    mx = fmax(mx, d);
  }
  for (int o = 16; o > 0; o >>= 1) mx = fmax(mx, __shfl_xor_sync(0xffffffffu, mx, o));
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = mx;
  __syncthreads();
  if (threadIdx.x == 0) { for (int w = 1; w < (int)(blockDim.x >> 5); ++w) mx = fmax(mx, red[w]); fmx[f] = mx; }
}

__global__ void __launch_bounds__(1024) k_ogate_mean(const double* __restrict__ db, const double* __restrict__ fmx, const int* __restrict__ n_valid, int n,
                                                    int frames, int nb, double top_db, double threshold_db, double* __restrict__ power, int* __restrict__ status) {
  __shared__ double scratch[32];
  if (n_valid && *n_valid < n) { if (threadIdx.x == 0) { *power = 0.0; *status = 0; } return; }
  double mx = -1e300;
  for (int f = 0; f < frames; ++f) mx = fmax(mx, fmx[f]);
  const double floor_db = mx - top_db;
  double part = 0.0;
  const size_t total = (size_t)frames * nb;
  for (size_t i = threadIdx.x; i < total; i += blockDim.x) { const double d = db[i]; part += d > floor_db ? d : floor_db; }
  const double sum = block_sum(part, scratch);
  if (threadIdx.x == 0) {
    const double pw = sum / (double)total;
    *power = pw;
    *status = pw < -threshold_db ? 2 : 1;              // 1: chunk passes, 2: chunk is silent (the reference sends None)
  }
}

int output_gate_frames(int n, int hop) { return 1 + n / hop; }
size_t output_gate_scratch_doubles(int n, int n_fft, int hop) { return (size_t)output_gate_frames(n, hop) * (n_fft / 2 + 1 + 1); }

// Stream-ordered, device pointers.  d_n_valid (may be null): the gate only runs when *d_n_valid >= n (else status 0).
int output_gate_async(Engine* e, const double* d_wave, const int* d_n_valid, int n, int n_fft, int hop, double threshold_db,
                      double* d_scratch, double* d_power, int* d_status, cudaStream_t st) {
  RYK_CHECK(n_fft >= 64 && n_fft <= kTwiddleN && (n_fft & (n_fft - 1)) == 0, "unsupported STFT size for the output gate");
  RYK_CHECK(n > n_fft / 2, "output chunk too short for a reflect-centred STFT");
  static bool attr_set = false;
  if (!attr_set) { RYK_CUDA(cudaFuncSetAttribute(k_ogate_stft, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(sizeof(double2) * kTwiddleN))); attr_set = true; }
  const int frames = output_gate_frames(n, hop), nb = n_fft / 2 + 1;
  double* d_db = d_scratch;
  double* d_fmax = d_scratch + (size_t)frames * nb;
  k_ogate_stft<<<frames, 256, sizeof(double2) * n_fft, st>>>(d_wave, d_n_valid, n, n_fft, hop, 1e-10, d_db, d_fmax, e->d_twiddle);
  k_ogate_mean<<<1, 1024, 0, st>>>(d_db, d_fmax, d_n_valid, n, frames, nb, 80.0, threshold_db, d_power, d_status);
  RYK_CUDA(cudaGetLastError());
  return 0;
}

}  // namespace ryk
