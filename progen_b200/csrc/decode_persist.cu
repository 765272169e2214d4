// KV-cached autoregressive decode as ONE persistent kernel (BASELINE config 5; reference utils.py:106-135, sample.py:66-71).
//
// One cooperative kernel (one CTA per SM) generates every position of the launch, with no kernel launch between its
// steps: the phases of a layer (LN + shift + QKV + rotary + cache | windowed attention | out-proj + residual | LN + shift +
// FF-in + GLU/GELU | [gMLP: gate LN + causal spatial mix | SGU proj] | FF-out + residual) are separated by a grid barrier
// (one atomic + one acquire poll per CTA), and the token loop, the sampler and the position counter stay on the device: no
// host round trip.  Sampler 0 is the reference's (top-k filter that keeps k-1 and zeroes the rest, Gumbel-max over host
// noise, `seq[pos+1] += id` — quirks Q5/Q6); sampler 1 is the standard one (top-k, temperature, nucleus, in-kernel Philox
// Gumbel noise, per-token log-probabilities, and an early exit once every sequence has sampled EOS).
//
// A position is ~65 dependent phases, so single-stream speed is LATENCY: a barrier is arrive -> prefetch -> wait, and between
// the atomic and the poll every warp requests what does not depend on the other CTAs' output of the phase: its slice of the
// NEXT GEMV phase's weights (registers), biases, LN scales, rotary entries, the residual values it will add to (offsets and
// rows come from per-launch tables).  What is left on the critical path is one L2 round trip for the activations, two block
// reductions (LN), the FMAs, a 9-shuffle reduction and the barrier itself.
//
// BATCH: `B` sequences advance in lock step ([B, 1] rows per step) and the step streams the weights ONCE for all of them.
// B <= 8: a lane holds 8 weights of two rows and multiplies them with every staged activation row (reduction over lanes).
// B > 8, bf16 weights: tensor pipe — the CTA's weight slice goes to shared memory as bf16, every fp32 activation is split into
// three bf16 terms (8 + 8 + 8 mantissa bits) and mma.sync.m16n8k16 accumulates the exact products in fp32; activations arrive by
// bulk copies, LayerNorm rows are normalised in shared memory.  B > 8, fp32 weights: lane = sequence, weights broadcast from
// shared memory.  More than 32 sequences: the 32-sequence tile runs twice per phase on the same staged weights.
// Sequence b samples position p+1 iff p+1 >= start[b] (its prime is kept before).
#include "common.cuh"
#include "tc_ptx.cuh"
#include "../../include/progen_b200.h"
#include <cmath>
#include <type_traits>

namespace {

using namespace tc;

constexpr int WSEGS = 32;               // (row pair, 256-column segment) weight units of one CTA per wave
constexpr int MAXEV = 160;              // profile events per sampled CTA (grid barriers of one step)
constexpr int MAXSPLIT = 8;             // SGU: most splits of the history range
// threads per CTA, every batch tile.  A single sequence is a latency chain: 8 warps are enough.  For B > 8 the phases are
// bound by L2 traffic of the activation staging and by memory latency, not by issue slots, so 512 threads are no faster.
constexpr int TPB = 256;
constexpr int WPB = TPB / 32;
constexpr int MAXSEG = WSEGS / WPB;     // units a warp holds in registers

template <int BT, bool TCW = false> struct Tile {   // shared-memory geometry by batch tile; TCW: bf16 weights on the tensor pipe (BT > 8)
  static constexpr bool LANEB = BT > 8;                       // whole-batch formulations (B > 8)
  static constexpr bool TC = LANEB && TCW;
  static constexpr int KCB = BT == 1 ? 8192 : (BT <= 8 ? 2048 : 512);   // activation columns staged per pass
  // row pitch of the staged activations: +4 floats -> conflict-free float4 per lane (lane = sequence); +8 -> conflict-free
  // 8-byte A-fragment loads of mma.m16n8k16 (lane = (row, column pair))
  static constexpr int XP = TC ? KCB + 8 : (LANEB ? KCB + 4 : KCB);
  static constexpr int BTP = BT | 1;                          // odd row pitch of the partial-sum scratch
  static constexpr int STATF = (2 * BT + 2 * WPB + 3) & ~3;   // LN statistics [BT][2] + two block-reduction scratches
  // one wave's weights: fp32 [2 * PW rows][256 * KS] (lane = sequence), or bf16 [rows][256 * KS + 8] (tensor pipe)
  static constexpr int WSM = TC ? WSEGS * 256 + 2 * WSEGS * 4 : (LANEB ? WSEGS * 512 : 0);
  static constexpr int NMT = LANEB ? BT / 16 : 1;             // TC: 16-sequence m-tiles; warp = (m-tile, K split)
  static constexpr int NKH = LANEB ? WPB / NMT : 1;
  // partial sums: K segments (B <= 8) | accumulators of the upper half of the K splits, halved round by round (tensor pipe) |
  // none (lane = sequence)
  static constexpr int PART = TC ? (NKH / 2) * NMT * 32 * 32 : (LANEB ? 0 : WSEGS * 2 * BTP);
  static constexpr int NBG = LANEB ? BT / 32 : 1;             // lane = sequence: 32-sequence groups; warp = (group, row split)
  static constexpr int NRQ = WPB / NBG;
  static constexpr int MAXLP = (WSEGS + NRQ - 1) / NRQ;       // pairs of a wave per row split
};

static __device__ __forceinline__ void mma_bf16_16816(float (&c)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
               : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
               : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
// fp32 pair -> three bf16 pairs whose sum is the fp32 value to 2^-24 (8 + 8 + 8 mantissa bits): with bf16 weights every
// product is exact in the fp32 accumulator, so the tensor pipe computes the same sums as the fp32 FMA path up to order
static __device__ __forceinline__ void split3_bf16x2(float x0, float x1, uint32_t& h1, uint32_t& h2, uint32_t& h3) {
  h1 = pack_bf16x2(x0, x1);
  const float r0 = x0 - __uint_as_float(h1 << 16), r1 = x1 - __uint_as_float(h1 & 0xffff0000u);
  h2 = pack_bf16x2(r0, r1);
  const float q0 = r0 - __uint_as_float(h2 << 16), q1 = r1 - __uint_as_float(h2 & 0xffff0000u);
  h3 = pack_bf16x2(q0, q1);
}

// ------------------------------------------------------------------------------------------------ grid barrier
// monotonic counter: every CTA adds 1, then polls until all gridDim.x arrivals of this round are in.  `prof` (optional):
// CTA 0 and the last CTA record clock64 at entry and exit of every barrier of the launch's LAST step.
struct Prof { long long* buf; int ev; bool on; };
// CTA 0, thread 0: clock64 at point k (< 8) inside the phase that ends with barrier number pf.ev  (buf + 4 * MAXEV: [MAXEV][8])
static __device__ __forceinline__ void prof_mark(const Prof& pf, int k) {
  if (pf.on && blockIdx.x == 0 && threadIdx.x == 0 && pf.ev < MAXEV) pf.buf[4 * MAXEV + pf.ev * 8 + k] = clock64();
}
static __device__ __forceinline__ void grid_arrive(unsigned int* bar, unsigned int& round, Prof& pf, long long& t0) {
  __syncthreads();
  if (threadIdx.x == 0) {
    if (pf.on) t0 = clock64();
    ++round;
    __threadfence();
    atomicAdd(bar, 1u);
  }
}
static __device__ __forceinline__ void grid_wait(unsigned int* bar, unsigned int round, Prof& pf, long long t0) {
  if (threadIdx.x == 0) {
    const unsigned int target = round * gridDim.x;
    unsigned int v;
    do {
      asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(bar) : "memory");
    } while (v < target);
    if (pf.on && pf.ev < MAXEV) {
      long long* e = pf.buf + ((blockIdx.x == 0 ? 0 : 1) * MAXEV + pf.ev) * 2;
      e[0] = t0; e[1] = clock64();
      ++pf.ev;
    }
  }
  __syncthreads();
}
static __device__ __forceinline__ void grid_sync(unsigned int* bar, unsigned int& round, Prof& pf) {
  long long t0 = 0;
  grid_arrive(bar, round, pf, t0);
  grid_wait(bar, round, pf, t0);
}

// 8 consecutive weights of a row as one lane's registers: bf16 = one 16-byte load, fp32 = two
template <typename TW> struct W8 { uint4 q[sizeof(TW) / 2]; };
template <typename TW> static __device__ __forceinline__ void w8_load(W8<TW>& w, const TW* p) {
#pragma unroll
  for (int i = 0; i < (int)(sizeof(TW) / 2); ++i) w.q[i] = __ldg(reinterpret_cast<const uint4*>(p) + i);
}
template <typename TW> static __device__ __forceinline__ void w8_zero(W8<TW>& w) {
#pragma unroll
  for (int i = 0; i < (int)(sizeof(TW) / 2); ++i) w.q[i] = make_uint4(0u, 0u, 0u, 0u);
}
static __device__ __forceinline__ void w8_unpack(const W8<bf16>& w, float (&f)[8]) {
  const uint32_t u[4] = {w.q[0].x, w.q[0].y, w.q[0].z, w.q[0].w};
#pragma unroll
  for (int i = 0; i < 4; ++i) { f[2 * i] = __uint_as_float(u[i] << 16); f[2 * i + 1] = __uint_as_float(u[i] & 0xffff0000u); }
}
static __device__ __forceinline__ void w8_unpack(const W8<float>& w, float (&f)[8]) {
  f[0] = __uint_as_float(w.q[0].x); f[1] = __uint_as_float(w.q[0].y); f[2] = __uint_as_float(w.q[0].z); f[3] = __uint_as_float(w.q[0].w);
  f[4] = __uint_as_float(w.q[1].x); f[5] = __uint_as_float(w.q[1].y); f[6] = __uint_as_float(w.q[1].z); f[7] = __uint_as_float(w.q[1].w);
}
template <typename TW> struct WRegs { W8<TW> a[MAXSEG], c[MAXSEG]; int pl[MAXSEG], ks[MAXSEG]; };   // + each unit's (pair, K segment) in its wave

enum { EP_BIAS = 0, EP_ROTARY_CACHE = 1, EP_RESIDUAL = 2, EP_GLU = 3, EP_GELU = 4 };
enum { PRO_NONE = 0, PRO_LN = 1, PRO_ATT = 2, PRO_SGU = 3 };

// CTA c owns the output row PAIRS [c*P/G, (c+1)*P/G) of a GEMV phase, cut along K into 256-column segments; a wave is PW pairs
// x KS segments <= WSEGS slots, slot s -> warp s % WPB, unit s / WPB of that warp
struct Geo { int p_lo, np, KS, PW, nwaves; };
struct Phase {
  const void* wt;          // [N(,x2 for GLU), K]
  const float* bias;       // [N] or null
  const float* xin;        // [B, ldx] input rows
  int ldx;
  float* out;              // [B, ldo]
  int ldo;
  int N, K;
  int epi;
  // prologue
  int pro;                 // PRO_LN: x <- shift(LN(x) * scale); PRO_ATT: x <- merged attention partials (B = 1);
                           // PRO_SGU: x <- xin * sum of the SGU partial gates
  const float* ln_scale;
  float* ln_prev;          // [B][2][K/2] token-shift state (read [pos&1], write [(pos+1)&1]); null: no shift
  const float* aux;        // PRO_ATT: att_part; PRO_SGU: partial gates [nsplit][B][K]
  int window, nsplit;
  long long aux_stride;    // PRO_SGU: elements between two splits' partial gates (total sequences x K)
  // rotary / cache epilogue
  float* kcache; float* vcache; int inner, dim_head, n;
  const float* rot_sin; const float* rot_cos;
  int pos;
  Geo g;                   // this CTA's share (filled when the table is built)
};

// values a thread needs in a phase that do NOT depend on the previous phase: loaded before the barrier (BT == 1 only)
struct Pre { float b0, b1, o0, o1, sn, cs; float4 sc, pv; float* d0; float* d1; };   // d0 / d1: where the pair's two results go

// Work split of one GEMV phase: CTA c owns the output row PAIRS [c*P/G, (c+1)*P/G) (pair = rows 2p, 2p+1, or p, p+N for
// GLU), cut along K into 256-column segments; a wave is PW pairs x KS segments <= WSEGS slots, slot s -> warp s % WPB.
static __device__ __forceinline__ Geo make_geo(const Phase& ph) {
  const int npairs = ph.epi == EP_GLU ? ph.N : ph.N >> 1;
  Geo g;
  g.p_lo = (int)(blockIdx.x * (unsigned)npairs / gridDim.x);              // npairs <= 8192, grid <= a few hundred: 32 bits
  g.np = (int)((blockIdx.x + 1) * (unsigned)npairs / gridDim.x) - g.p_lo;
  g.KS = (ph.K + 255) >> 8;
  g.PW = WSEGS / g.KS;
  g.nwaves = (g.np + g.PW - 1) / g.PW;
  return g;
}

// Issue the 16-byte loads of one wave's weights (no use of the data here: the caller may put a grid barrier and other
// phases between this and the FMAs, so HBM / L2 latency overlaps the barrier).
template <typename TW>
static __device__ __forceinline__ void load_wave(const Phase& ph, const Geo& g, int wave, WRegs<TW>& w) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const TW* W = reinterpret_cast<const TW*>(ph.wt);
  const int pbase = wave * g.PW;
  const int pw = min(g.PW, g.np - pbase);
#pragma unroll
  for (int i = 0; i < MAXSEG; ++i) {
    const int sw = warp + WPB * i;
    const int pl = sw / g.KS, ks = sw - pl * g.KS;
    const int k = ks * 256 + lane * 8;
    w.pl[i] = pl; w.ks[i] = ks;
    if (pl < pw && k < ph.K) {
      const int pair = g.p_lo + pbase + pl;
      const long long r0 = ph.epi == EP_GLU ? pair : 2 * pair, r1 = ph.epi == EP_GLU ? pair + ph.N : 2 * pair + 1;
      w8_load<TW>(w.a[i], W + r0 * ph.K + k);
      w8_load<TW>(w.c[i], W + r1 * ph.K + k);
    } else {
      w8_zero<TW>(w.a[i]);
      w8_zero<TW>(w.c[i]);
    }
  }
}

// Single stream: what a warp / a finalizing thread needs of wave 0 of a phase, precomputed once per launch — the prefetch runs
// between a barrier's arrive and wait on every warp, so its instruction count (divisions by runtime values, 64-bit offsets) is
// phase time whenever it exceeds the barrier's own latency.
struct __align__(16) UnitEnt { int off0, off1; short pl, ks; int kmax; };   // weight offsets of the unit's two rows (-1: no unit), columns left in its segment
struct FinEnt { int r0, r1, d0, sel, rj; };                    // rows, store offset (sel: 0 out, 1 K cache, 2 V cache), rotary index
// the finalizer entry of `pair` (single stream: built into the unit tables, or in the prefetch when they do not fit)
static __device__ __forceinline__ FinEnt fin_entry(const Phase& ph, int pair) {
  FinEnt f;
  f.r0 = ph.epi == EP_GLU ? pair : 2 * pair; f.r1 = ph.epi == EP_GLU ? pair + ph.N : 2 * pair + 1;
  f.d0 = f.r0; f.sel = 0; f.rj = 0;
  if (ph.epi == EP_ROTARY_CACHE) {
    const int sec = f.r0 / ph.inner, c = f.r0 % ph.inner;
    f.rj = (f.r0 % ph.dim_head) >> 1;
    f.sel = sec;
    f.d0 = sec == 0 ? c : (c / ph.dim_head) * ph.n * ph.dim_head + c % ph.dim_head;
  }
  return f;
}
static __device__ void build_unit_tables(const Phase& ph, UnitEnt* ut, FinEnt* ft, int u /* 0 .. WSEGS-1 */) {
  const Geo& g = ph.g;
  const int pw = min(g.PW, g.np);
  {
    const int pl = u / g.KS, ks = u - pl * g.KS;
    UnitEnt e;
    e.pl = (short)pl; e.ks = (short)ks; e.kmax = ph.K - ks * 256; e.off0 = e.off1 = -1;
    if (pl < pw && e.kmax > 0) {
      const int pair = g.p_lo + pl;
      const int r0 = ph.epi == EP_GLU ? pair : 2 * pair, r1 = ph.epi == EP_GLU ? pair + ph.N : 2 * pair + 1;
      e.off0 = r0 * ph.K + ks * 256; e.off1 = r1 * ph.K + ks * 256;
    }
    ut[u] = e;
  }
  ft[u] = u < pw ? fin_entry(ph, g.p_lo + u) : FinEnt{0, 0, 0, 0, 0};
}

// everything of phase `ph` (pos filled in) that can be loaded before the barrier in front of it.  ut / ft: this phase's
// precomputed tables (single stream), or null
template <int BT, typename TW>
static __device__ __forceinline__ void prefetch_phase(const Phase& ph, WRegs<TW>& w, Pre& pre, const UnitEnt* ut, const FinEnt* ft) {
  const Geo& g = ph.g;
  if constexpr (BT == 1) {
    const int t = threadIdx.x, lane = t & 31, warp = t >> 5;
    if (ut != nullptr) {
      const TW* W = reinterpret_cast<const TW*>(ph.wt);
#pragma unroll
      for (int i = 0; i < MAXSEG; ++i) {
        const UnitEnt u = ut[warp + WPB * i];
        w.pl[i] = u.pl; w.ks[i] = u.ks;
        if (u.off0 >= 0 && lane * 8 < u.kmax) {
          w8_load<TW>(w.a[i], W + u.off0 + lane * 8);
          w8_load<TW>(w.c[i], W + u.off1 + lane * 8);
        } else {
          w8_zero<TW>(w.a[i]);
          w8_zero<TW>(w.c[i]);
        }
      }
    } else {
      load_wave<TW>(ph, g, 0, w);                                // (deep models: the per-launch tables do not fit shared memory)
    }
    if (t < min(g.PW, g.np)) {                                  // this thread finalizes pair t of wave 0
      const FinEnt f = ft != nullptr ? ft[t] : fin_entry(ph, g.p_lo + t);
      pre.b0 = ph.bias ? ph.bias[f.r0] : 0.f;
      pre.b1 = ph.bias ? ph.bias[f.r1] : 0.f;
      pre.d0 = ph.out + f.r0; pre.d1 = ph.out + f.r1;
      if (ph.epi == EP_RESIDUAL) { pre.o0 = __ldcg(ph.out + f.r0); pre.o1 = __ldcg(ph.out + f.r1); }
      if (ph.epi == EP_ROTARY_CACHE) {
        const int hd = ph.dim_head >> 1;
        pre.sn = ph.rot_sin[ph.pos * hd + f.rj]; pre.cs = ph.rot_cos[ph.pos * hd + f.rj];
        pre.d0 = (f.sel == 0 ? ph.out : (f.sel == 1 ? ph.kcache : ph.vcache) + ph.pos * ph.dim_head) + f.d0;
        pre.d1 = pre.d0 + 1;
      }
    }
    const int k = t * 4;
    if (ph.pro == PRO_LN && k < ph.K && ph.K <= 4 * TPB) {
      pre.sc = *reinterpret_cast<const float4*>(ph.ln_scale + k);
      if (ph.ln_prev && k < (ph.K >> 1)) pre.pv = __ldcg(reinterpret_cast<const float4*>(ph.ln_prev + (ph.pos & 1) * (ph.K >> 1) + k));
    }
  } else {
    load_wave<TW>(ph, g, 0, w);
  }
}

static __device__ __forceinline__ float block_sum(float v, float* scratch /* [WPB] */) {
  v = warp_sum(v);
  if ((threadIdx.x & 31) == 0) scratch[threadIdx.x >> 5] = v;
  __syncthreads();
  float t = 0.f;
#pragma unroll
  for (int k = 0; k < WPB; ++k) t += scratch[k];
  return t;
}

// shared-memory position of activation column k (k % 4 == 0) of a staged row.  B <= 8: the two 16-byte halves of every
// 8-column group live in two planes, so the lanes of a warp (8 columns each) read consecutive 16-byte words.
template <int BT> static __device__ __forceinline__ int xs_off(int k) {
  if constexpr (Tile<BT>::LANEB) return k;
  else return ((k >> 2) & 1) * (Tile<BT>::KCB / 2) + (k >> 3) * 4;
}

// merged attention output of (sequence 0, columns k..k+3) from the per-slice partials (B = 1: the out-proj phase merges)
static __device__ __forceinline__ float4 merge_att(const Phase& ph, int k) {
  const int dh = ph.dim_head, w = ph.window;
  const int win = ph.pos / w, i = ph.pos % w;
  const int nreal = (win > 0 ? w : 0) + i + 1;
  const int nsl = (nreal + 31) / 32;
  const int KS = (2 * w + 31) / 32;
  const float* pb = ph.aux + (long long)(k / dh) * KS * (dh + 4);
  const int c = k % dh;
  float M = win == 0 ? 0.f : -INFINITY;               // zero look-back keys of window 0: logit 0 (quirk Q1)
  float Lt = 0.f;
  float4 a = make_float4(0.f, 0.f, 0.f, 0.f);
  for (int s0 = 0; s0 < nsl; s0 += 8) {
    float2 ml[8];
    float4 o[8];
#pragma unroll
    for (int u = 0; u < 8; ++u) {
      const bool on = s0 + u < nsl;
      const float* pk = pb + (on ? s0 + u : 0) * (dh + 4);
      ml[u] = __ldcg(reinterpret_cast<const float2*>(pk));
      o[u] = __ldcg(reinterpret_cast<const float4*>(pk + 4 + c));
      if (!on) ml[u] = make_float2(-INFINITY, 0.f);        // weight exp(-inf) = 0
    }
    float Mn = M;
#pragma unroll
    for (int u = 0; u < 8; ++u) Mn = fmaxf(Mn, ml[u].x);
    const float fo = (M == -INFINITY) ? 0.f : expf(M - Mn);
    Lt *= fo; a.x *= fo; a.y *= fo; a.z *= fo; a.w *= fo;
    M = Mn;
#pragma unroll
    for (int u = 0; u < 8; ++u) {
      const float f = expf(ml[u].x - M);
      Lt = fmaf(ml[u].y, f, Lt);
      a.x = fmaf(f, o[u].x, a.x); a.y = fmaf(f, o[u].y, a.y); a.z = fmaf(f, o[u].z, a.z); a.w = fmaf(f, o[u].w, a.w);
    }
  }
  if (win == 0) Lt += (float)w * expf(-M);
  const float inv = 1.f / Lt;
  return make_float4(a.x * inv, a.y * inv, a.z * inv, a.w * inv);
}

// One GEMV / skinny-GEMM phase over all B sequences.  BT = compile-time batch tile (B <= BT).  `w`, `pre` hold what
// prefetch_phase loaded for THIS phase (the caller ran it before the previous grid barrier, or just now).
// SLOT (the queue kernels): sequence b is at position spos[b] (shared memory) instead of the shared ph.pos.
template <int BT, typename TW, bool SLOT = false>
static __device__ __forceinline__ void gemv_phase(const Phase& ph, int B, float* xs, float* part, float* stat, float* wsm, WRegs<TW>& w, const Pre& pre, const Prof& pf,
                                           uint32_t sbar, uint32_t& sparity, bool reload_w0 = false, const int* spos = nullptr) {
  using TL = Tile<BT, sizeof(TW) == 2>;
  constexpr int KCB = TL::KCB, XP = TL::XP, BTP = TL::BTP;
  constexpr bool LANEB = TL::LANEB, TC = TL::TC;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const Geo g = ph.g;
  auto pos_of = [&](int b) -> int {
    if constexpr (SLOT) return spos[b];
    else return ph.pos;
  };
  const int nchunks = (ph.K + KCB - 1) / KCB;
  const int half = ph.K >> 1;
  bool staged = false;
  bool wsm_ready = false;
  if constexpr (TC) {
    // tensor pipe: wave 0's weights (prefetched registers) go to shared memory first — nothing of it depends on the
    // activations, so it overlaps their copy instead of following the LayerNorm (the previous phase's / pass's readers of wsm
    // are behind a CTA barrier already)
    if (!(reload_w0 && g.nwaves > 1)) {
      const int WKP = g.KS * 256 + 8;
      __nv_bfloat16* wb = reinterpret_cast<__nv_bfloat16*>(wsm);
#pragma unroll
      for (int i = 0; i < MAXSEG; ++i) {
        const int pl = w.pl[i], ks = w.ks[i];
        if (pl >= g.PW) continue;
        __nv_bfloat16* d0 = wb + (2 * pl) * WKP + ks * 256 + lane * 8;
        *reinterpret_cast<uint4*>(d0) = w.a[i].q[0];
        *reinterpret_cast<uint4*>(d0 + WKP) = w.c[i].q[0];
      }
      wsm_ready = true;
    }
  }
  if (BT == 1 && ph.K <= 4 * TPB) {
    // single sequence, one float4 per thread: LN statistics, scale, token shift and the staging in one pass
    const int k = threadIdx.x * 4;
    const bool in = k < ph.K;
    float4 t = make_float4(0.f, 0.f, 0.f, 0.f);
    if (in) {
      if (ph.pro == PRO_ATT) t = merge_att(ph, k);
      else t = __ldcg(reinterpret_cast<const float4*>(ph.xin + k));
    }
    if (ph.pro == PRO_SGU && in) {
      float4 gsum = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
      for (int s = 0; s < MAXSPLIT; ++s) {
        if (s < ph.nsplit) {
          const float4 v = __ldcg(reinterpret_cast<const float4*>(ph.aux + s * ph.aux_stride + k));
          gsum.x += v.x; gsum.y += v.y; gsum.z += v.z; gsum.w += v.w;
        }
      }
      t.x *= gsum.x; t.y *= gsum.y; t.z *= gsum.z; t.w *= gsum.w;
    }
    if (ph.pro == PRO_LN) {
      const float mean = block_sum((t.x + t.y) + (t.z + t.w), stat + 2 * BT) / ph.K;
      prof_mark(pf, 5);
      const float a0 = t.x - mean, a1 = t.y - mean, a2 = t.z - mean, a3 = t.w - mean;
      const float q = block_sum(in ? (a0 * a0 + a1 * a1) + (a2 * a2 + a3 * a3) : 0.f, stat + 2 * BT + WPB);
      prof_mark(pf, 6);
      const float rstd = rsqrtf(q / ph.K + 1e-5f);
      if (in) {
        t.x = a0 * rstd * pre.sc.x; t.y = a1 * rstd * pre.sc.y; t.z = a2 * rstd * pre.sc.z; t.w = a3 * rstd * pre.sc.w;
        if (ph.ln_prev && k < half) {
          if (blockIdx.x == 0) *reinterpret_cast<float4*>(ph.ln_prev + ((ph.pos + 1) & 1) * half + k) = t;
          t = pre.pv;
        }
      }
    }
    if (in) *reinterpret_cast<float4*>(xs + xs_off<BT>(k)) = t;
    __syncthreads();
    staged = true;
  } else if (LANEB && ph.pro == PRO_LN && nchunks == 1 && ph.K <= 512 && (ph.K & 127) == 0) {
    // B > 8: the rows arrive by bulk copies (L2 -> shared memory at the L2 rate: every CTA reads the same 128 KB at the same
    // time), the token-shift state of this warp's rows by register loads issued before the wait; then a warp per row normalises
    // in place.  Instruction count matters here (64 rows per CTA): NJ = K / 128 is a compile-time constant, 1 / K a multiply.
    constexpr int RPW = (BT + WPB - 1) / WPB;               // rows per warp
    fence_proxy_async();
    __syncthreads();
    if (threadIdx.x == 0) mbar_expect_tx(sbar, (uint32_t)(B * ph.K * 4));
    if (threadIdx.x < B)
      asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                   ::"r"(smem_u32(xs + threadIdx.x * XP)), "l"(ph.xin + (long long)threadIdx.x * ph.ldx), "r"((uint32_t)(ph.K * 4)), "r"(sbar) : "memory");
    float4 pvv[RPW][2];
#pragma unroll
    for (int rr = 0; rr < RPW; ++rr) {
      const int b = warp + rr * WPB;
#pragma unroll
      for (int j = 0; j < 2; ++j) {
        const int k = j * 128 + lane * 4;
        pvv[rr][j] = (ph.ln_prev && b < B && k < half)
                         ? __ldcg(reinterpret_cast<const float4*>(ph.ln_prev + (long long)b * ph.K + (pos_of(b) & 1) * half + k)) : make_float4(0.f, 0.f, 0.f, 0.f);
      }
    }
    const float inv_k = 1.f / (float)ph.K;
    mbar_wait(sbar, sparity);
    sparity ^= 1u;
    prof_mark(pf, 7);
    auto norm_rows = [&](auto nj_c) {
      constexpr int NJ = decltype(nj_c)::value;
      float4 sc[NJ];
#pragma unroll
      for (int j = 0; j < NJ; ++j) sc[j] = *reinterpret_cast<const float4*>(ph.ln_scale + j * 128 + lane * 4);
#pragma unroll
      for (int r0 = 0; r0 < RPW; r0 += 2) {
        // two rows in flight per warp (their reductions are independent chains)
        float4 v[2][NJ];
        float mean[2], rstd[2];
#pragma unroll
        for (int u = 0; u < 2; ++u) {
          const int b = warp + (r0 + u) * WPB;
          const float* xr = xs + (b < B ? b : 0) * XP + lane * 4;
#pragma unroll
          for (int j = 0; j < NJ; ++j) v[u][j] = *reinterpret_cast<const float4*>(xr + j * 128);
        }
        {
          float sa = 0.f, sb = 0.f;
#pragma unroll
          for (int j = 0; j < NJ; ++j) { sa += (v[0][j].x + v[0][j].y) + (v[0][j].z + v[0][j].w); sb += (v[1][j].x + v[1][j].y) + (v[1][j].z + v[1][j].w); }
#pragma unroll
          for (int off = 16; off > 0; off >>= 1) { sa += __shfl_xor_sync(0xffffffffu, sa, off); sb += __shfl_xor_sync(0xffffffffu, sb, off); }
          mean[0] = sa * inv_k; mean[1] = sb * inv_k;
          float qa = 0.f, qb = 0.f;
#pragma unroll
          for (int j = 0; j < NJ; ++j) {
            v[0][j].x -= mean[0]; v[0][j].y -= mean[0]; v[0][j].z -= mean[0]; v[0][j].w -= mean[0];
            v[1][j].x -= mean[1]; v[1][j].y -= mean[1]; v[1][j].z -= mean[1]; v[1][j].w -= mean[1];
            qa = fmaf(v[0][j].x, v[0][j].x, fmaf(v[0][j].y, v[0][j].y, fmaf(v[0][j].z, v[0][j].z, fmaf(v[0][j].w, v[0][j].w, qa))));
            qb = fmaf(v[1][j].x, v[1][j].x, fmaf(v[1][j].y, v[1][j].y, fmaf(v[1][j].z, v[1][j].z, fmaf(v[1][j].w, v[1][j].w, qb))));
          }
#pragma unroll
          for (int off = 16; off > 0; off >>= 1) { qa += __shfl_xor_sync(0xffffffffu, qa, off); qb += __shfl_xor_sync(0xffffffffu, qb, off); }
          rstd[0] = rsqrtf(qa * inv_k + 1e-5f); rstd[1] = rsqrtf(qb * inv_k + 1e-5f);
        }
#pragma unroll
        for (int u = 0; u < 2; ++u) {
          const int rr = r0 + u;
          const int b = warp + rr * WPB;
          if (rr >= RPW || b >= B) continue;                 // warp-uniform
          float* xr = xs + b * XP + lane * 4;
          float* st = ph.ln_prev ? ph.ln_prev + (long long)b * ph.K + ((pos_of(b) + 1) & 1) * half + lane * 4 : nullptr;
#pragma unroll
          for (int j = 0; j < NJ; ++j) {
            float4 t = make_float4(v[u][j].x * rstd[u] * sc[j].x, v[u][j].y * rstd[u] * sc[j].y, v[u][j].z * rstd[u] * sc[j].z, v[u][j].w * rstd[u] * sc[j].w);
            if (st && j * 128 + lane * 4 < half) {           // (half = NJ * 64: j < NJ / 2, or the lower lanes of the middle j)
              if (blockIdx.x == 0) *reinterpret_cast<float4*>(st + j * 128) = t;
              t = pvv[rr < RPW ? rr : 0][j < 2 ? j : 0];
            }
            *reinterpret_cast<float4*>(xr + j * 128) = t;
          }
        }
      }
    };
    switch (ph.K >> 7) {
      case 1: norm_rows(std::integral_constant<int, 1>{}); break;
      case 2: norm_rows(std::integral_constant<int, 2>{}); break;
      case 3: norm_rows(std::integral_constant<int, 3>{}); break;
      default: norm_rows(std::integral_constant<int, 4>{}); break;
    }
    __syncthreads();
    staged = true;
  } else if (BT > 1 && ph.pro == PRO_LN && nchunks == 1 && ph.K <= 1024) {
    // whole rows fit one pass: warp per sequence, the row stays in registers between the statistics and the staging;
    // RF rows (NJ float4 per lane each) in flight per warp
    auto ln_rows = [&](auto rf_c, auto nj_c) {
      constexpr int RF = decltype(rf_c)::value, NJ = decltype(nj_c)::value;
      for (int b0 = warp; b0 < B; b0 += RF * WPB) {
        float4 v[RF][NJ], pvv[RF][NJ / 2];                  // the rows and their token-shift state (first half of the columns)
#pragma unroll
        for (int rr = 0; rr < RF; ++rr) {
          const int b = b0 + rr * WPB;
#pragma unroll
          for (int j = 0; j < NJ; ++j) {
            const int k = j * 128 + lane * 4;
            v[rr][j] = (b < B && k < ph.K) ? __ldcg(reinterpret_cast<const float4*>(ph.xin + (long long)b * ph.ldx + k)) : make_float4(0.f, 0.f, 0.f, 0.f);
          }
#pragma unroll
          for (int j = 0; j < NJ / 2; ++j) {
            const int k = j * 128 + lane * 4;
            pvv[rr][j] = (ph.ln_prev && b < B && k < half)
                             ? __ldcg(reinterpret_cast<const float4*>(ph.ln_prev + (long long)b * ph.K + (pos_of(b) & 1) * half + k)) : make_float4(0.f, 0.f, 0.f, 0.f);
          }
        }
#pragma unroll
        for (int rr = 0; rr < RF; ++rr) {
          const int b = b0 + rr * WPB;
          if (b >= B) continue;
          float s = 0.f;
#pragma unroll
          for (int j = 0; j < NJ; ++j) s += (v[rr][j].x + v[rr][j].y) + (v[rr][j].z + v[rr][j].w);
          const float mean = warp_sum(s) / ph.K;
          float q = 0.f;
#pragma unroll
          for (int j = 0; j < NJ; ++j) {
            if (j * 128 + lane * 4 < ph.K) {
              const float a0 = v[rr][j].x - mean, a1 = v[rr][j].y - mean, a2 = v[rr][j].z - mean, a3 = v[rr][j].w - mean;
              q += (a0 * a0 + a1 * a1) + (a2 * a2 + a3 * a3);
            }
          }
          const float rstd = rsqrtf(warp_sum(q) / ph.K + 1e-5f);
          float* st = ph.ln_prev ? ph.ln_prev + (long long)b * ph.K : nullptr;       // [2][K/2]
#pragma unroll
          for (int j = 0; j < NJ; ++j) {
            const int k = j * 128 + lane * 4;
            if (k < ph.K) {
              const float4 sc = *reinterpret_cast<const float4*>(ph.ln_scale + k);
              float4 t;
              t.x = (v[rr][j].x - mean) * rstd * sc.x; t.y = (v[rr][j].y - mean) * rstd * sc.y;
              t.z = (v[rr][j].z - mean) * rstd * sc.z; t.w = (v[rr][j].w - mean) * rstd * sc.w;
              if (st && k < half) {                         // k < half  =>  j < NJ / 2 (half = K / 2 <= NJ * 64)
                if (blockIdx.x == 0) *reinterpret_cast<float4*>(st + ((pos_of(b) + 1) & 1) * half + k) = t;
                t = pvv[rr][j < NJ / 2 ? j : 0];
              }
              *reinterpret_cast<float4*>(xs + b * XP + xs_off<BT>(k)) = t;
            }
          }
        }
      }
    };
    constexpr int RFW = 4;
    if (ph.K <= 512) ln_rows(std::integral_constant<int, RFW>{}, std::integral_constant<int, 4>{});
    else ln_rows(std::integral_constant<int, RFW / 2>{}, std::integral_constant<int, 8>{});
    __syncthreads();
    staged = true;
  } else if (ph.pro == PRO_LN) {
    // LN statistics of every sequence's row (whole K), once per phase: warp b % WPB handles row b
    for (int b = warp; b < B; b += WPB) {
      const float* xr = ph.xin + (long long)b * ph.ldx;
      float s = 0.f;
      for (int k = lane * 4; k < ph.K; k += 128) { const float4 t = __ldcg(reinterpret_cast<const float4*>(xr + k)); s += (t.x + t.y) + (t.z + t.w); }
      s = warp_sum(s);
      const float mean = s / ph.K;
      float q = 0.f;
      for (int k = lane * 4; k < ph.K; k += 128) {
        const float4 t = __ldcg(reinterpret_cast<const float4*>(xr + k));
        const float a0 = t.x - mean, a1 = t.y - mean, a2 = t.z - mean, a3 = t.w - mean;
        q += (a0 * a0 + a1 * a1) + (a2 * a2 + a3 * a3);
      }
      q = warp_sum(q);
      if (lane == 0) { stat[2 * b] = mean; stat[2 * b + 1] = rsqrtf(q / ph.K + 1e-5f); }
    }
    __syncthreads();
  }
  // stage x[:, k0 .. k0+kn) (with the prologue) into shared memory; U independent loads in flight per thread
  constexpr int U = LANEB ? 8 : 4;
  auto stage_regs = [&](int kc) {
    const int k0 = kc * KCB, kn = min(KCB, ph.K - k0);
    const int nvec = B * (kn >> 2);
    for (int base = 0; base < nvec; base += U * TPB) {
      float4 t[U];
#pragma unroll
      for (int u = 0; u < U; ++u) {
        const int idx = min(base + u * TPB + (int)threadIdx.x, nvec - 1);       // clamped: the load is unconditional
        const int b = idx / (kn >> 2), k = (idx % (kn >> 2)) * 4;
        t[u] = __ldcg(reinterpret_cast<const float4*>(ph.xin + (long long)b * ph.ldx + k0 + k));
      }
#pragma unroll
      for (int u = 0; u < U; ++u) {
        const int idx = base + u * TPB + threadIdx.x;
        if (idx >= nvec) continue;
        const int b = idx / (kn >> 2), k = (idx % (kn >> 2)) * 4;
        float4 v = t[u];
        if (ph.pro == PRO_LN) {
          const float mean = stat[2 * b], rstd = stat[2 * b + 1];
          const float4 sc = *reinterpret_cast<const float4*>(ph.ln_scale + k0 + k);
          v.x = (v.x - mean) * rstd * sc.x; v.y = (v.y - mean) * rstd * sc.y;
          v.z = (v.z - mean) * rstd * sc.z; v.w = (v.w - mean) * rstd * sc.w;
          if (ph.ln_prev && k0 + k < half) {
            float* st = ph.ln_prev + (long long)b * ph.K;            // [2][K/2]
            const float4 pv = __ldcg(reinterpret_cast<const float4*>(st + (pos_of(b) & 1) * half + k0 + k));
            if (blockIdx.x == 0) *reinterpret_cast<float4*>(st + ((pos_of(b) + 1) & 1) * half + k0 + k) = v;
            v = pv;
          }
        }
        *reinterpret_cast<float4*>(xs + b * XP + xs_off<BT>(k)) = v;
      }
    }
  };
  // PRO_SGU: x = xs * (sum of the partial gates); the activations and split 0's gate are loaded together
  auto stage_sgu = [&](int kc) {
    constexpr int U2 = LANEB ? 8 : 4;
    const int k0 = kc * KCB, kn = min(KCB, ph.K - k0);
    const int nvec = B * (kn >> 2);
    for (int base = 0; base < nvec; base += U2 * TPB) {
      float4 t[U2], gq[U2];
#pragma unroll
      for (int u = 0; u < U2; ++u) {
        const int idx = min(base + u * TPB + (int)threadIdx.x, nvec - 1);
        const int b = idx / (kn >> 2), k = (idx % (kn >> 2)) * 4;
        t[u] = __ldcg(reinterpret_cast<const float4*>(ph.xin + (long long)b * ph.ldx + k0 + k));
        gq[u] = __ldcg(reinterpret_cast<const float4*>(ph.aux + (long long)b * ph.K + k0 + k));
      }
#pragma unroll
      for (int u = 0; u < U2; ++u) {
        const int idx = base + u * TPB + threadIdx.x;
        if (idx >= nvec) continue;
        const int b = idx / (kn >> 2), k = (idx % (kn >> 2)) * 4;
        float4 gsum = gq[u];
        for (int sp = 1; sp < ph.nsplit; ++sp) {
          const float4 q = __ldcg(reinterpret_cast<const float4*>(ph.aux + sp * ph.aux_stride + (long long)b * ph.K + k0 + k));
          gsum.x += q.x; gsum.y += q.y; gsum.z += q.z; gsum.w += q.w;
        }
        *reinterpret_cast<float4*>(xs + b * XP + xs_off<BT>(k)) = make_float4(t[u].x * gsum.x, t[u].y * gsum.y, t[u].z * gsum.z, t[u].w * gsum.w);
      }
    }
  };
  // B > 8, no prologue: one bulk copy (L2 -> shared memory, no registers, no L1) per sequence row
  auto stage = [&](int kc) {
    if (LANEB && ph.pro == PRO_NONE) {
      const int k0 = kc * KCB, kn = min(KCB, ph.K - k0);
      fence_proxy_async();                                  // earlier generic accesses to xs are ordered before the async writes
      __syncthreads();
      if (threadIdx.x == 0) mbar_expect_tx(sbar, (uint32_t)(B * kn * 4));
      if (threadIdx.x < B) {
        asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                     ::"r"(smem_u32(xs + threadIdx.x * XP)), "l"(ph.xin + (long long)threadIdx.x * ph.ldx + k0), "r"((uint32_t)(kn * 4)), "r"(sbar) : "memory");
      }
      mbar_wait(sbar, sparity);
      sparity ^= 1u;
    } else if (ph.pro == PRO_SGU) {
      stage_sgu(kc);
    } else {
      stage_regs(kc);
    }
  };
  // bias + activation / residual / rotary + cache for the two rows of `pair` of sequence b
  auto epilogue = [&](int b, int pair, float s0, float s1) {
    const int r0 = ph.epi == EP_GLU ? pair : 2 * pair, r1 = ph.epi == EP_GLU ? pair + ph.N : 2 * pair + 1;
    if (ph.bias) { s0 += ph.bias[r0]; s1 += ph.bias[r1]; }
    float* o = ph.out + (long long)b * ph.ldo;
    if (ph.epi == EP_BIAS) { o[r0] = s0; o[r1] = s1; }
    else if (ph.epi == EP_RESIDUAL) { o[r0] = __ldcg(o + r0) + s0; o[r1] = __ldcg(o + r1) + s1; }
    else if (ph.epi == EP_GELU) { o[r0] = gelu_tanh(s0); o[r1] = gelu_tanh(s1); }
    else if (ph.epi == EP_GLU) { o[r0] = s0 * gelu_tanh(s1); }
    else {  // EP_ROTARY_CACHE: rotary on q, k AND v (progen.py:87); k, v rows go to the caches at position pos
      const int hd = ph.dim_head >> 1, j = (r0 % ph.dim_head) >> 1, p = pos_of(b);
      const float sn = ph.rot_sin[p * hd + j], cs = ph.rot_cos[p * hd + j];
      const float o0 = s0 * cs - s1 * sn, o1 = s1 * cs + s0 * sn;
      const int sec = r0 / ph.inner, c = r0 % ph.inner;
      float* dst = sec == 0 ? o + c
                            : (sec == 1 ? ph.kcache : ph.vcache) + (((long long)b * (ph.inner / ph.dim_head) + c / ph.dim_head) * ph.n + p) * ph.dim_head + c % ph.dim_head;
      dst[0] = o0; dst[1] = o1;
    }
  };
  if (!staged && nchunks == 1) { stage(0); __syncthreads(); }
  prof_mark(pf, 1);
  for (int wave = 0; wave < g.nwaves; ++wave) {
    if (wave > 0 || (reload_w0 && g.nwaves > 1)) load_wave<TW>(ph, g, wave, w);   // (a later sub-batch of a multi-wave phase: `w` holds the last wave)
    const int pbase = wave * g.PW;
    const int pw = min(g.PW, g.np - pbase);
    if constexpr (!LANEB) {
      for (int kc = 0; kc < nchunks; ++kc) {
        if (nchunks > 1) { __syncthreads(); stage(kc); __syncthreads(); }
        const int k0 = kc * KCB;
        float red0[MAXSEG], red1[MAXSEG];                 // BT == 1: the units' lane-partial sums, reduced together below
#pragma unroll
        for (int i = 0; i < MAXSEG; ++i) {
          red0[i] = 0.f; red1[i] = 0.f;
          const int sw = warp + WPB * i;
          const int pl = w.pl[i], ks = w.ks[i];
          const int kseg = ks * 256;
          if (pl >= pw || kseg < k0 || kseg >= k0 + KCB) continue;     // warp-uniform
          const int k = kseg + lane * 8;
          float acc0[BT], acc1[BT];
#pragma unroll
          for (int b = 0; b < BT; ++b) { acc0[b] = 0.f; acc1[b] = 0.f; }
          if (k < ph.K) {
            float a[8], c[8];
            w8_unpack(w.a[i], a);
            w8_unpack(w.c[i], c);
            const float* xk = xs + xs_off<BT>(k - k0);
#pragma unroll
            for (int b = 0; b < BT; ++b) {
              if (b < B) {
                const float4 x0 = *reinterpret_cast<const float4*>(xk + b * XP);
                const float4 x1 = *reinterpret_cast<const float4*>(xk + b * XP + KCB / 2);
                acc0[b] = fmaf(a[0], x0.x, fmaf(a[1], x0.y, fmaf(a[2], x0.z, fmaf(a[3], x0.w, acc0[b]))));
                acc0[b] = fmaf(a[4], x1.x, fmaf(a[5], x1.y, fmaf(a[6], x1.z, fmaf(a[7], x1.w, acc0[b]))));
                acc1[b] = fmaf(c[0], x0.x, fmaf(c[1], x0.y, fmaf(c[2], x0.z, fmaf(c[3], x0.w, acc1[b]))));
                acc1[b] = fmaf(c[4], x1.x, fmaf(c[5], x1.y, fmaf(c[6], x1.z, fmaf(c[7], x1.w, acc1[b]))));
              }
            }
          }
          if constexpr (BT == 1) {
            red0[i] = acc0[0]; red1[i] = acc1[0];
          } else {
            // reduce over lanes: lane b ends with sequence b's sums
            float* p0 = part + (sw * 2) * BTP;
            float s0 = 0.f, s1 = 0.f;
#pragma unroll
            for (int j = 0; j < BT; ++j) {
              const float t0 = warp_sum(acc0[j]), t1 = warp_sum(acc1[j]);
              if (lane == j) { s0 = t0; s1 = t1; }
            }
            if (lane < BT) { p0[lane] = s0; p0[BTP + lane] = s1; }
          }
        }
        if constexpr (BT == 1) {
          // 2 * MAXSEG values per lane -> transposing butterfly: 4 + 2 + 1 exchanges leave value j in the lanes with
          // (lane & 7) == j summed over their group of 8, two more sum the four groups (9 shuffles instead of 40)
          static_assert(MAXSEG == 4, "the reduction below is written for 8 values");
          float v[8] = {red0[0], red1[0], red0[1], red1[1], red0[2], red1[2], red0[3], red1[3]};
#pragma unroll
          for (int H = 4; H >= 1; H >>= 1) {
            const bool up = (lane & H) != 0;
#pragma unroll
            for (int j = 0; j < H; ++j) {
              const float send = up ? v[j] : v[j + H];
              const float keep = up ? v[j + H] : v[j];
              v[j] = keep + __shfl_xor_sync(0xffffffffu, send, H);
            }
          }
          float tot = v[0];
          tot += __shfl_xor_sync(0xffffffffu, tot, 8);
          tot += __shfl_xor_sync(0xffffffffu, tot, 16);
          // lane j < 8 holds value j = unit (j >> 1), row (j & 1) -> part[(warp + WPB * unit) * 2 + row]   (BTP == 1)
          if (lane < 8) part[(warp + WPB * (lane >> 1)) * 2 + (lane & 1)] = tot;
        }
      }
      __syncthreads();
      prof_mark(pf, 2);
      // finalize this wave's pairs: sum the K segments in order, then the epilogue (threads run over pairs fastest, so
      // the two adjacent output columns of neighbouring pairs coalesce)
      if (BT == 1 && wave == 0) {
        // this thread's pair, its operands and store addresses were prepared before the barrier (prefetch_phase)
        const int pl = threadIdx.x;
        if (pl < pw) {
          float s0 = pre.b0, s1 = pre.b1;
          for (int ks = 0; ks < g.KS; ++ks) { s0 += part[(pl * g.KS + ks) * 2]; s1 += part[(pl * g.KS + ks) * 2 + 1]; }
          if (ph.epi == EP_BIAS) { *pre.d0 = s0; *pre.d1 = s1; }
          else if (ph.epi == EP_RESIDUAL) { *pre.d0 = pre.o0 + s0; *pre.d1 = pre.o1 + s1; }
          else if (ph.epi == EP_GELU) { *pre.d0 = gelu_tanh(s0); *pre.d1 = gelu_tanh(s1); }
          else if (ph.epi == EP_GLU) { *pre.d0 = s0 * gelu_tanh(s1); }
          else { *pre.d0 = s0 * pre.cs - s1 * pre.sn; *pre.d1 = s1 * pre.cs + s0 * pre.sn; }
        }
      } else {
        for (int idx = threadIdx.x; idx < pw * B; idx += TPB) {
          const int b = idx / pw, pl = idx - b * pw;
          float s0 = 0.f, s1 = 0.f;
          for (int ks = 0; ks < g.KS; ++ks) {
            const float* pp = part + ((pl * g.KS + ks) * 2) * BTP + b;
            s0 += pp[0]; s1 += pp[BTP];
          }
          epilogue(b, g.p_lo + pbase + pl, s0, s1);
        }
      }
      if (wave + 1 < g.nwaves) __syncthreads();
    } else {
      if constexpr (TC) {
        // ---- tensor pipe (bf16 weights).  (1) this wave's weights -> shared memory as they are: bf16 [row = 2*pl + which][WK + 8]
        constexpr int NMT = TL::NMT, NKH = TL::NKH, NTMAX = 2 * WSEGS / 8;
        const int WK = g.KS * 256, WKP = WK + 8;               // +8 bf16: the 8 rows of a B fragment land in distinct banks
        __nv_bfloat16* wb = reinterpret_cast<__nv_bfloat16*>(wsm);
        if (!(wave == 0 && wsm_ready)) {                       // (wave 0 was written at the top of the phase, under the activation copies)
          __syncthreads();                                     // the previous wave's readers of wsm are done
#pragma unroll
          for (int i = 0; i < MAXSEG; ++i) {
            const int pl = w.pl[i], ks = w.ks[i];
            if (pl >= g.PW) continue;
            __nv_bfloat16* d0 = wb + (2 * pl) * WKP + ks * 256 + lane * 8;
            *reinterpret_cast<uint4*>(d0) = w.a[i].q[0];
            *reinterpret_cast<uint4*>(d0 + WKP) = w.c[i].q[0];
          }
        }
        // (2) warp = (m-tile of 16 sequences, K split): C[16 x 8 per n-tile] += A[16 x 16](x, three bf16 terms) B[16 x 8](weights)
        const int mt = warp % NMT, kh = warp / NMT;
        const int NT = (2 * pw + 7) >> 3;                      // n-tiles of 8 weight rows
        const int gr = lane >> 2, gc = (lane & 3) * 2;
        float acc[NTMAX][4];
#pragma unroll
        for (int nt = 0; nt < NTMAX; ++nt) { acc[nt][0] = acc[nt][1] = acc[nt][2] = acc[nt][3] = 0.f; }
        // epilogue operands of n-tiles n0, n0 + 1 for this lane's two sequences (b0, b0 + 8) and pair 4 nt + (lane & 3)
        const int b0 = mt * 16 + gr;
        constexpr int NRH = SLOT ? 2 : 1;                      // rotary entries per (n-tile, sequence): the two sequences' positions differ
        auto load_ops = [&](int n0, float (&bia)[2][2], float (&old)[2][4], float (&rot)[2][NRH][2]) {
#pragma unroll
          for (int u = 0; u < 2; ++u) {
            const int nt = n0 + u;
            const int pl = nt * 4 + (lane & 3);
            const bool v = nt < NT && pl < pw;
            const int pair = g.p_lo + pbase + (v ? pl : 0);
            const int r0 = ph.epi == EP_GLU ? pair : 2 * pair, r1 = ph.epi == EP_GLU ? pair + ph.N : 2 * pair + 1;
            bia[u][0] = ph.bias ? ph.bias[r0] : 0.f;
            bia[u][1] = ph.bias ? ph.bias[r1] : 0.f;
            old[u][0] = old[u][1] = old[u][2] = old[u][3] = 0.f;
            if (ph.epi == EP_RESIDUAL) {
              const float* o0 = ph.out + (long long)(b0 < B ? b0 : 0) * ph.ldo;
              const float* o1 = ph.out + (long long)(b0 + 8 < B ? b0 + 8 : 0) * ph.ldo;
              old[u][0] = __ldcg(o0 + r0); old[u][1] = __ldcg(o0 + r1);
              old[u][2] = __ldcg(o1 + r0); old[u][3] = __ldcg(o1 + r1);
            }
#pragma unroll
            for (int hb = 0; hb < NRH; ++hb) {
              rot[u][hb][0] = rot[u][hb][1] = 0.f;
              if (ph.epi == EP_ROTARY_CACHE) {
                const int hd = ph.dim_head >> 1, j = (r0 % ph.dim_head) >> 1;
                const int p = pos_of(b0 + 8 * hb < B ? b0 + 8 * hb : 0);
                rot[u][hb][0] = ph.rot_sin[p * hd + j]; rot[u][hb][1] = ph.rot_cos[p * hd + j];
              }
            }
          }
        };
        float bia0[2][2], old0[2][4], rot0[2][NRH][2];
        load_ops(0, bia0, old0, rot0);                         // in flight under the MMA loop (every warp: kh is only known to be 0 later)
        for (int kc = 0; kc < nchunks; ++kc) {
          __syncthreads();                                     // wsm written (kc == 0) / the previous chunk's xs readers done
          if (kc == 0) prof_mark(pf, 5);
          if (nchunks > 1) { stage(kc); __syncthreads(); }
          const int k0 = kc * KCB, kn = min(KCB, ph.K - k0);
          const float* xa = xs + (mt * 16 + gr) * XP + gc;
          // the k-loop is instantiated for 1, 2, 4 or 8 n-tiles: fragment loads and MMAs of absent tiles cost issue slots,
          // and issue slots are what bounds this loop (the three-way split is ~50 instructions per k-step on its own)
          auto mma_chunk = [&](auto ntc_c) {
            constexpr int NTC = decltype(ntc_c)::value;
#pragma unroll 2
            for (int kb = kh * 16; kb < kn; kb += NKH * 16) {
              uint32_t a1[4], a2[4], a3[4];
              {
                const float2 v0 = *reinterpret_cast<const float2*>(xa + kb);
                const float2 v1 = *reinterpret_cast<const float2*>(xa + 8 * XP + kb);
                const float2 v2 = *reinterpret_cast<const float2*>(xa + kb + 8);
                const float2 v3 = *reinterpret_cast<const float2*>(xa + 8 * XP + kb + 8);
                split3_bf16x2(v0.x, v0.y, a1[0], a2[0], a3[0]);
                split3_bf16x2(v1.x, v1.y, a1[1], a2[1], a3[1]);
                split3_bf16x2(v2.x, v2.y, a1[2], a2[2], a3[2]);
                split3_bf16x2(v3.x, v3.y, a1[3], a2[3], a3[3]);
              }
              const __nv_bfloat16* wk = wb + k0 + kb + gc;
              uint32_t fb0[NTC], fb1[NTC];
#pragma unroll
              for (int nt = 0; nt < NTC; ++nt) {
                // row of the staged slice this lane's fragment column comes from; clamped to the 2 * PW rows that exist (wide K:
                // PW < 4, i.e. fewer than 8 rows — columns past them belong to no pair and are dropped by the epilogue)
                const int row = min((nt < NT ? nt : 0) * 8 + gr, 2 * g.PW - 1);
                fb0[nt] = *reinterpret_cast<const uint32_t*>(wk + row * WKP);
                fb1[nt] = *reinterpret_cast<const uint32_t*>(wk + row * WKP + 8);
              }
              // term-major, smallest terms first: consecutive MMAs hit different accumulators
#pragma unroll
              for (int nt = 0; nt < NTC; ++nt) if (nt < NT) mma_bf16_16816(acc[nt], a3, fb0[nt], fb1[nt]);
#pragma unroll
              for (int nt = 0; nt < NTC; ++nt) if (nt < NT) mma_bf16_16816(acc[nt], a2, fb0[nt], fb1[nt]);
#pragma unroll
              for (int nt = 0; nt < NTC; ++nt) if (nt < NT) mma_bf16_16816(acc[nt], a1, fb0[nt], fb1[nt]);
            }
          };
          if (NT <= 1) mma_chunk(std::integral_constant<int, 1>{});
          else if (NT <= 2) mma_chunk(std::integral_constant<int, 2>{});
          else if (NT <= 4) mma_chunk(std::integral_constant<int, 4>{});
          else mma_chunk(std::integral_constant<int, NTMAX>{});
        }
        prof_mark(pf, 6);
        // (3) the K splits are summed pairwise, halving round by round through shared memory (split q + h -> split q, a fixed
        // order), then split 0 runs the epilogue from its registers: lane holds (sequence gr | gr + 8 of the m-tile) x (weight
        // rows 8 nt + gc, + 1 = the two rows of pair 4 nt + gc / 2)
#pragma unroll
        for (int h = NKH / 2; h >= 1; h >>= 1) {
          if (kh >= h && kh < 2 * h) {
#pragma unroll
            for (int nt = 0; nt < NTMAX; ++nt)
              if (nt < NT) *reinterpret_cast<float4*>(part + ((kh - h) * NMT + mt) * 1024 + nt * 128 + lane * 4) =
                  make_float4(acc[nt][0], acc[nt][1], acc[nt][2], acc[nt][3]);
          }
          __syncthreads();
          if (kh < h) {
#pragma unroll
            for (int nt = 0; nt < NTMAX; ++nt) {
              if (nt < NT) {
                const float4 v = *reinterpret_cast<const float4*>(part + (kh * NMT + mt) * 1024 + nt * 128 + lane * 4);
                acc[nt][0] += v.x; acc[nt][1] += v.y; acc[nt][2] += v.z; acc[nt][3] += v.w;
              }
            }
          }
          if (h > 1) __syncthreads();
        }
        prof_mark(pf, 2);
        if (kh == 0) {
          // two n-tiles at a time: every operand of their epilogues first (bias, old residual values, rotary entries:
          // independent loads; those of the first two n-tiles were requested before the MMA loop), then the math and the stores
#pragma unroll
          for (int n0 = 0; n0 < NTMAX; n0 += 2) {
            if (n0 >= NT) continue;                            // (no break: the loop must unroll, acc[] is indexed statically)
            float bia[2][2], old[2][4], rot[2][NRH][2];
            if (n0 == 0) {
#pragma unroll
              for (int u = 0; u < 2; ++u) {
                bia[u][0] = bia0[u][0]; bia[u][1] = bia0[u][1];
#pragma unroll
                for (int hb = 0; hb < NRH; ++hb) { rot[u][hb][0] = rot0[u][hb][0]; rot[u][hb][1] = rot0[u][hb][1]; }
                old[u][0] = old0[u][0]; old[u][1] = old0[u][1]; old[u][2] = old0[u][2]; old[u][3] = old0[u][3];
              }
            } else {
              load_ops(n0, bia, old, rot);
            }
#pragma unroll
            for (int u = 0; u < 2; ++u) {
              const int nt = n0 + u;
              const int pl = nt * 4 + (lane & 3);
              if (nt < NT && pl < pw) {
                const int pair = g.p_lo + pbase + pl;
                const int r0 = ph.epi == EP_GLU ? pair : 2 * pair, r1 = ph.epi == EP_GLU ? pair + ph.N : 2 * pair + 1;
#pragma unroll
                for (int hb = 0; hb < 2; ++hb) {
                  const int b = b0 + 8 * hb;
                  if (b >= B) continue;
                  const float s0 = acc[nt][2 * hb] + bia[u][0], s1 = acc[nt][2 * hb + 1] + bia[u][1];
                  float* o = ph.out + (long long)b * ph.ldo;
                  if (ph.epi == EP_BIAS) { o[r0] = s0; o[r1] = s1; }
                  else if (ph.epi == EP_RESIDUAL) { o[r0] = old[u][2 * hb] + s0; o[r1] = old[u][2 * hb + 1] + s1; }
                  else if (ph.epi == EP_GELU) { o[r0] = gelu_tanh(s0); o[r1] = gelu_tanh(s1); }
                  else if (ph.epi == EP_GLU) { o[r0] = s0 * gelu_tanh(s1); }
                  else {
                    const float sn = rot[u][SLOT ? hb : 0][0], cs = rot[u][SLOT ? hb : 0][1];
                    const int sec = r0 / ph.inner, c = r0 % ph.inner;
                    float* dst = sec == 0 ? o + c : (sec == 1 ? ph.kcache : ph.vcache) + (((long long)b * (ph.inner / ph.dim_head) + c / ph.dim_head) * ph.n + pos_of(b)) * ph.dim_head + c % ph.dim_head;
                    dst[0] = s0 * cs - s1 * sn; dst[1] = s1 * cs + s0 * sn;
                  }
                }
              }
            }
          }
        }
      } else {
      // ---- lane = sequence.  (1) this wave's weights -> shared memory as fp32 [row = 2*pl + which][256*KS columns]
      constexpr int NBG = TL::NBG, NRQ = TL::NRQ, MAXLP = TL::MAXLP;
      const int WK = g.KS * 256;                             // columns per staged row (tail zero-filled by load_wave)
      __syncthreads();                                       // the previous wave's / phase's readers of wsm are done
#pragma unroll
      for (int i = 0; i < MAXSEG; ++i) {
        const int pl = w.pl[i], ks = w.ks[i];
        if (pl >= g.PW) continue;
        float a[8], c[8];
        w8_unpack(w.a[i], a);
        w8_unpack(w.c[i], c);
        float* d0 = wsm + (2 * pl) * WK + ks * 256 + lane * 8;
        *reinterpret_cast<float4*>(d0) = make_float4(a[0], a[1], a[2], a[3]);
        *reinterpret_cast<float4*>(d0 + 4) = make_float4(a[4], a[5], a[6], a[7]);
        *reinterpret_cast<float4*>(d0 + WK) = make_float4(c[0], c[1], c[2], c[3]);
        *reinterpret_cast<float4*>(d0 + WK + 4) = make_float4(c[4], c[5], c[6], c[7]);
      }
      // (2) warp = (32-sequence group, row split q): pairs q, q + NRQ, ... of the wave; 32 activations of the lane's
      // sequence in registers against the warp's rows, weights by broadcast loads
      const int bg = warp % NBG, q = warp / NBG;
      const int b = bg * 32 + lane;
      float acc[MAXLP][2][2];
#pragma unroll
      for (int lp = 0; lp < MAXLP; ++lp) { acc[lp][0][0] = acc[lp][0][1] = acc[lp][1][0] = acc[lp][1][1] = 0.f; }
      for (int kc = 0; kc < nchunks; ++kc) {
        __syncthreads();                                     // wsm written (kc == 0) / the previous chunk's xs readers done
        if (nchunks > 1) { stage(kc); __syncthreads(); }
        const int k0 = kc * KCB, kn = min(KCB, ph.K - k0);
        const float* xrow = xs + (b < B ? b : 0) * XP;
        for (int kb = 0; kb < kn; kb += 32) {
          float x[32];
#pragma unroll
          for (int j = 0; j < 8; ++j) {
            const float4 t = *reinterpret_cast<const float4*>(xrow + kb + j * 4);
            x[4 * j] = t.x; x[4 * j + 1] = t.y; x[4 * j + 2] = t.z; x[4 * j + 3] = t.w;
          }
          const float* wk = wsm + k0 + kb;
#pragma unroll
          for (int lp = 0; lp < MAXLP; ++lp) {
            const int pl = q + NRQ * lp;
            if (pl < pw) {                                   // warp-uniform
#pragma unroll
              for (int wh = 0; wh < 2; ++wh) {
                const float* wr = wk + (2 * pl + wh) * WK;
                float e0 = acc[lp][wh][0], e1 = acc[lp][wh][1];
#pragma unroll
                for (int j = 0; j < 8; j += 2) {
                  const float4 u0 = *reinterpret_cast<const float4*>(wr + j * 4);        // same address in every lane: broadcast
                  const float4 u1 = *reinterpret_cast<const float4*>(wr + j * 4 + 4);
                  e0 = fmaf(u0.x, x[4 * j], fmaf(u0.y, x[4 * j + 1], fmaf(u0.z, x[4 * j + 2], fmaf(u0.w, x[4 * j + 3], e0))));
                  e1 = fmaf(u1.x, x[4 * j + 4], fmaf(u1.y, x[4 * j + 5], fmaf(u1.z, x[4 * j + 6], fmaf(u1.w, x[4 * j + 7], e1))));
                }
                acc[lp][wh][0] = e0; acc[lp][wh][1] = e1;
              }
            }
          }
        }
      }
      // (3) epilogue straight from the registers (lane = sequence)
      if (b < B) {
#pragma unroll
        for (int lp = 0; lp < MAXLP; ++lp) {
          const int pl = q + NRQ * lp;
          if (pl < pw) epilogue(b, g.p_lo + pbase + pl, acc[lp][0][0] + acc[lp][0][1], acc[lp][1][0] + acc[lp][1][1]);
        }
      }
      }
    }
  }
}

// ------------------------------------------------------------------------------------------------ attention
// task = (sequence, head, slice of 32 keys), one warp: partial (m, l, o[dh]) -> att_part[(b, head)][slice][dh + 4].  All of
// the task's K and V loads are independent of each other (lane = key for the logits; lane = (key group, 4 channels) for
// the value sum), so a task is ONE memory round trip.  The out-proj phase merges the partials (plus window 0's w zero keys
// with logit 0, quirk Q1) while it stages its input (merge_att).  Single sequence only; B > 1 uses attention_batch.
template <int NL /* lanes that cover one value row with float4 = dim_head / 4 */>
static __device__ void attention_phase_t(const progen_decode_run_t& r, const float* kcache, const float* vcache, int pos, float* sq /* smem [WPB][dh] */) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int dh = r.dim_head, w = r.window, I = r.inner;
  const int win = pos / w, i = pos % w;
  const int key0 = win > 0 ? (win - 1) * w : 0;
  const int nreal = (win > 0 ? w : 0) + i + 1;
  const int nsl = (nreal + 31) / 32;
  const int KS = (2 * w + 31) / 32;                         // slots per (b, head) in att_part
  const int PS = dh + 4;                                    // floats per slot: m, l, -, -, o[dh]
  const int tasks = r.B * r.heads * nsl;
  const float scale = rsqrtf((float)dh);
  constexpr int KG = 32 / NL;                               // key groups
  constexpr int NH = NL >= 2 ? NL / 2 : 1;                  // value quads per lane and batch of loads
  const int kg = lane / NL, c4 = (lane % NL) * 4;
  float* q_s = sq + warp * dh;
  for (int t = warp * gridDim.x + blockIdx.x; t < tasks; t += gridDim.x * WPB) {
    const int sl = t % nsl, bh = t / nsl, hh = bh % r.heads, b = bh / r.heads;
    const float* qv = r.q + (long long)b * I + hh * dh;
    __syncwarp();
    if (lane < NL) *reinterpret_cast<float4*>(q_s + lane * 4) = __ldcg(reinterpret_cast<const float4*>(qv + lane * 4));
    const int j = sl * 32 + lane;
    const bool valid = j < nreal;
    const int nk = min(32, nreal - sl * 32);
    const float* kr = kcache + (((long long)b * r.heads + hh) * r.n + key0 + (valid ? j : 0)) * dh;      // caches: [B][heads][n][dh]
    const float* vb = vcache + (((long long)b * r.heads + hh) * r.n + key0 + sl * 32) * dh + c4;
    // issue: the float4s of this lane's key row and the first half of this lane's value quads (keys kg, kg + KG, ...);
    // the second half goes out as soon as the key registers are consumed
    float4 kreg[NL], vreg[NH];
#pragma unroll
    for (int c = 0; c < NL; ++c) kreg[c] = __ldcg(reinterpret_cast<const float4*>(kr + c * 4));
#pragma unroll
    for (int jj = 0; jj < NH; ++jj) {
      const int key = kg + jj * KG;
      vreg[jj] = key < nk ? __ldcg(reinterpret_cast<const float4*>(vb + (long long)key * dh)) : make_float4(0.f, 0.f, 0.f, 0.f);
    }
    __syncwarp();
    float s = 0.f;
#pragma unroll
    for (int c = 0; c < NL; ++c) {
      const float4 qq = *reinterpret_cast<const float4*>(q_s + c * 4);
      s = fmaf(kreg[c].x, qq.x, s); s = fmaf(kreg[c].y, qq.y, s); s = fmaf(kreg[c].z, qq.z, s); s = fmaf(kreg[c].w, qq.w, s);
    }
    float4 vreg2[NH];
#pragma unroll
    for (int jj = 0; jj < NH; ++jj) {
      const int key = kg + (jj + NH) * KG;
      vreg2[jj] = (NH + jj < NL && key < nk) ? __ldcg(reinterpret_cast<const float4*>(vb + (long long)key * dh)) : make_float4(0.f, 0.f, 0.f, 0.f);
    }
    s = valid ? s * scale : -INFINITY;
    const float m = warp_max(s);
    const float p = valid ? expf(s - m) : 0.f;
    const float l = warp_sum(p);
    float4 o = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
    for (int jj = 0; jj < NL; ++jj) {
      const int key = kg + jj * KG;
      const float pj = __shfl_sync(0xffffffffu, p, key & 31);                  // p = 0 for keys past the slice's end
      const float4 vv = jj < NH ? vreg[jj % NH] : vreg2[jj % NH];
      o.x = fmaf(pj, vv.x, o.x); o.y = fmaf(pj, vv.y, o.y); o.z = fmaf(pj, vv.z, o.z); o.w = fmaf(pj, vv.w, o.w);
    }
    for (int off = NL; off < 32; off <<= 1) {
      o.x += __shfl_xor_sync(0xffffffffu, o.x, off); o.y += __shfl_xor_sync(0xffffffffu, o.y, off);
      o.z += __shfl_xor_sync(0xffffffffu, o.z, off); o.w += __shfl_xor_sync(0xffffffffu, o.w, off);
    }
    float* pt = r.att_part + ((long long)bh * KS + sl) * PS;
    if (lane < NL) *reinterpret_cast<float4*>(pt + 4 + lane * 4) = o;
    if (lane == 0) *reinterpret_cast<float2*>(pt) = make_float2(m, l);
  }
}

// B > 1: WP warps (1, 2, 4 or 8, all of one CTA) own one (sequence, head): each walks its share of the 16-key slices with a
// running (max, sum, out) and the WP partials are merged through shared memory — no global partials, no atomics, no fences.
// Two lanes per key for the logits (half a key row each: 32 registers at dim_head 64), lane = (key group, 4 channels) for
// the value sum; every load of a slice is independent of the others.
// PLAN: the number of sequences the work split is planned for (0: the launch's B; see run())
// SLOT (the queue kernels): sequence b is at position spos[b] (shared memory); the window of each (sequence, head) follows it
template <int NL, int PLAN, bool SLOT>
static __device__ void attention_batch_t(const progen_decode_run_t& r, const float* kcache, const float* vcache, int pos, float* sq /* smem >= WPB * (2 dh + 4) */,
                                         const int* spos) {
  static_assert(NL >= 2, "two lanes share a key row");
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  constexpr int dh = NL * 4, HK = NL / 2, KG = 32 / NL, NV = 16 / KG;
  const int w = r.window, I = r.inner;
  int win = pos / w, i = pos % w;
  int key0 = win > 0 ? (win - 1) * w : 0;
  int nreal = (win > 0 ? w : 0) + i + 1;
  int nsl = (nreal + 15) / 16;
  const int npairs = r.B * r.heads;
  int WP = 8;
  const int plan_pairs = PLAN > 0 ? PLAN * r.heads : npairs;
  while (WP > 1 && (long long)plan_pairs * WP > (long long)gridDim.x * WPB) WP >>= 1;
  const int slots = WPB / WP, slot = warp / WP, sub = warp % WP;
  const int rounds = (npairs + gridDim.x * slots - 1) / (gridDim.x * slots);
  const float scale = rsqrtf((float)dh);
  const int key_l = lane >> 1, hf = lane & 1;
  const int kg = lane / NL, c4 = (lane % NL) * 4;
  float* q_s = sq + warp * dh;                                // this warp's copy of q
  float* mrg = sq + WPB * dh;                                 // [WPB][dh + 4] partials
  for (int rnd = 0; rnd < rounds; ++rnd) {
    const int pr = (rnd * slots + slot) * gridDim.x + blockIdx.x;
    const bool on = pr < npairs;
    const int hh = on ? pr % r.heads : 0, b = on ? pr / r.heads : 0;
    float m = -INFINITY, lsum = 0.f;
    float4 o = make_float4(0.f, 0.f, 0.f, 0.f);
    if (on) {
      if constexpr (SLOT) {
        const int p = spos[b];
        win = p / w; i = p % w;
        key0 = win > 0 ? (win - 1) * w : 0;
        nreal = (win > 0 ? w : 0) + i + 1;
        nsl = (nreal + 15) / 16;
      }
      const float* qv = r.q + (long long)b * I + hh * dh;
      if (lane < NL) *reinterpret_cast<float4*>(q_s + lane * 4) = __ldcg(reinterpret_cast<const float4*>(qv + lane * 4));
      __syncwarp();
      const float* kbase = kcache + (((long long)b * r.heads + hh) * r.n + key0) * dh + hf * 4;   // lane hf takes float4s hf, hf + 2, ...:
                                                                                          // the pair reads one whole 32-byte sector per load
      const float* vbase = vcache + (((long long)b * r.heads + hh) * r.n + key0) * dh + c4;
      // two slices per iteration: all their loads are issued before the first use (one memory round trip for 32 keys), one
      // running-max update for both; a missing second slice re-reads the first with weight 0
      auto load_slice = [&](int sl, float4 (&kreg)[HK], float4 (&vreg)[NV]) {
        const int j = sl * 16 + key_l;
        const int nk = min(16, nreal - sl * 16);
        const float* kr = kbase + (long long)(j < nreal ? j : 0) * dh;
#pragma unroll
        for (int c = 0; c < HK; ++c) kreg[c] = __ldcg(reinterpret_cast<const float4*>(kr + c * 8));
#pragma unroll
        for (int jj = 0; jj < NV; ++jj) {
          const int key = kg + jj * KG;
          vreg[jj] = __ldcg(reinterpret_cast<const float4*>(vbase + (long long)(sl * 16 + (key < nk ? key : 0)) * dh));
        }
      };
      auto logit = [&](int sl, const float4 (&kreg)[HK], bool on2) {
        float s = 0.f;
#pragma unroll
        for (int c = 0; c < HK; ++c) {
          const float4 qq = *reinterpret_cast<const float4*>(q_s + hf * 4 + c * 8);
          s = fmaf(kreg[c].x, qq.x, s); s = fmaf(kreg[c].y, qq.y, s); s = fmaf(kreg[c].z, qq.z, s); s = fmaf(kreg[c].w, qq.w, s);
        }
        s += __shfl_xor_sync(0xffffffffu, s, 1);
        return (on2 && sl * 16 + key_l < nreal) ? s * scale : -INFINITY;
      };
      for (int sl = sub; sl < nsl; sl += 2 * WP) {
        const bool two = sl + WP < nsl;
        const int slb = two ? sl + WP : sl;
        float4 ka[HK], va[NV], kb[HK], vb[NV];
        load_slice(sl, ka, va);
        load_slice(slb, kb, vb);
        const float sa = logit(sl, ka, true), sb = logit(slb, kb, two);
        const float mn = fmaxf(m, warp_max(fmaxf(sa, sb)));   // finite: the first slice has at least one real key
        const float f = expf(m - mn);                          // 0 for the first iteration (m = -inf)
        const float pa = expf(sa - mn), pb = expf(sb - mn);    // exp(-inf) = 0 for masked keys
        lsum = lsum * f + (hf == 0 ? pa + pb : 0.f);           // each key once
        o.x *= f; o.y *= f; o.z *= f; o.w *= f;
        m = mn;
#pragma unroll
        for (int jj = 0; jj < NV; ++jj) {
          const int src = (2 * (kg + jj * KG)) & 31;           // (keys past the slice's end carry weight 0; their value row was clamped)
          const float ja = __shfl_sync(0xffffffffu, pa, src), jb = __shfl_sync(0xffffffffu, pb, src);
          o.x = fmaf(ja, va[jj].x, fmaf(jb, vb[jj].x, o.x)); o.y = fmaf(ja, va[jj].y, fmaf(jb, vb[jj].y, o.y));
          o.z = fmaf(ja, va[jj].z, fmaf(jb, vb[jj].z, o.z)); o.w = fmaf(ja, va[jj].w, fmaf(jb, vb[jj].w, o.w));
        }
      }
      for (int off = NL; off < 32; off <<= 1) {
        o.x += __shfl_xor_sync(0xffffffffu, o.x, off); o.y += __shfl_xor_sync(0xffffffffu, o.y, off);
        o.z += __shfl_xor_sync(0xffffffffu, o.z, off); o.w += __shfl_xor_sync(0xffffffffu, o.w, off);
      }
      lsum = warp_sum(lsum);
      float* pt = mrg + warp * (dh + 4);
      if (lane < NL) *reinterpret_cast<float4*>(pt + 4 + lane * 4) = o;
      if (lane == 0) { pt[0] = m; pt[1] = lsum; }
    }
    __syncthreads();
    if (on && sub == 0 && lane < NL) {
      // merge the WP partials (a warp with no slice left m = -inf, l = 0) plus window 0's w zero keys with logit 0 (quirk Q1)
      const float* pb = mrg + (slot * WP) * (dh + 4);
      float M = win == 0 ? 0.f : -INFINITY;
      for (int k = 0; k < WP; ++k) M = fmaxf(M, pb[k * (dh + 4)]);
      float Lt = win == 0 ? (float)w * expf(-M) : 0.f;
      float4 a = make_float4(0.f, 0.f, 0.f, 0.f);
      for (int k = 0; k < WP; ++k) {
        const float* pk = pb + k * (dh + 4);
        const float f = expf(pk[0] - M);
        Lt = fmaf(pk[1], f, Lt);
        const float4 ov = *reinterpret_cast<const float4*>(pk + 4 + lane * 4);
        a.x = fmaf(f, ov.x, a.x); a.y = fmaf(f, ov.y, a.y); a.z = fmaf(f, ov.z, a.z); a.w = fmaf(f, ov.w, a.w);
      }
      const float inv = 1.f / Lt;
      *reinterpret_cast<float4*>(r.att + (long long)b * I + hh * dh + lane * 4) = make_float4(a.x * inv, a.y * inv, a.z * inv, a.w * inv);
    }
    __syncthreads();
  }
}
template <int PLAN, bool SLOT>
static __device__ void attention_batch(const progen_decode_run_t& r, const float* kcache, const float* vcache, int pos, float* sq, const int* spos) {
  switch (r.dim_head) {
    case 64: attention_batch_t<16, PLAN, SLOT>(r, kcache, vcache, pos, sq, spos); break;
    case 32: attention_batch_t<8, PLAN, SLOT>(r, kcache, vcache, pos, sq, spos); break;
    case 16: attention_batch_t<4, PLAN, SLOT>(r, kcache, vcache, pos, sq, spos); break;
    default: attention_batch_t<2, PLAN, SLOT>(r, kcache, vcache, pos, sq, spos); break;
  }
}

static __device__ void attention_phase(const progen_decode_run_t& r, const float* kcache, const float* vcache, int pos, float* sq) {
  switch (r.dim_head) {
    case 64: attention_phase_t<16>(r, kcache, vcache, pos, sq); break;
    case 32: attention_phase_t<8>(r, kcache, vcache, pos, sq); break;
    case 16: attention_phase_t<4>(r, kcache, vcache, pos, sq); break;
    default: attention_phase_t<2>(r, kcache, vcache, pos, sq); break;
  }
}

// ------------------------------------------------------------------------------------------------ SGU (progen.py:166-184)
// a = gelu(proj_in) = [xs | gate] (C channels each).  gn = LN(gate) * scale -> history[b][pos]; gate' = sum_{k<=pos} W[pos,k]
// history[b][k] + bias[pos]; sg = xs * gate'.  Task = (sequence, block of 128 channels, split of the history range): the
// partial gate' goes to sg[split][b][c] (split 0 adds the current position's term and the bias); the SGU projection
// phase multiplies xs with the sum of the partials while it stages its input (PRO_SGU).
struct SguArgs { const float* ln_scale; const float* w; const float* b; float* hist; };
template <int PLAN>
static __device__ __forceinline__ int sgu_splits(const progen_decode_run_t& r) {
  const int base = (PLAN > 0 ? PLAN : r.B) * (r.hid / 2 / 128);
  int s = (int)gridDim.x / (base > 0 ? base : 1);
  return s < 1 ? 1 : (s > MAXSPLIT ? MAXSPLIT : s);
}
// SLOT (the queue kernels): sequence b is at position spos[b] (shared memory); its split boundaries follow that position
template <int PLAN, bool SLOT>
static __device__ void sgu_phase(const progen_decode_run_t& r, const SguArgs& L, int pos_, float* red /* smem [WPB][128] + stats */,
                                 const int* spos) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int C = r.hid / 2, n = r.n;
  const int cblocks = C / 128;
  const int S = sgu_splits<PLAN>(r);
  const int tasks = r.B * cblocks * S;
  float* stat = red + WPB * 128;
  for (int t = blockIdx.x; t < tasks; t += gridDim.x) {
    const int sp = t % S, cb = (t / S) % cblocks, b = t / (S * cblocks);
    int pos = pos_;
    if constexpr (SLOT) pos = spos[b];
    const int c0 = cb * 128 + lane * 4;
    float* hist = L.hist + (long long)b * n * C;
    const float* wrow = L.w + (long long)pos * n;
    const int k_lo = (int)((long long)pos * sp / S), k_hi = (int)((long long)pos * (sp + 1) / S);
    // history rows of this split, warps interleaved, 8 loads in flight per lane
    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
    for (int kb = k_lo + warp; kb < k_hi; kb += 8 * WPB) {
      float4 h[8];
      float wk[8];
#pragma unroll
      for (int u = 0; u < 8; ++u) {
        const int k = kb + u * WPB;
        if (k < k_hi) { wk[u] = __ldg(wrow + k); h[u] = __ldcg(reinterpret_cast<const float4*>(hist + (long long)k * C + c0)); }
      }
#pragma unroll
      for (int u = 0; u < 8; ++u) {
        if (kb + u * WPB < k_hi) {
          acc.x = fmaf(wk[u], h[u].x, acc.x); acc.y = fmaf(wk[u], h[u].y, acc.y); acc.z = fmaf(wk[u], h[u].z, acc.z); acc.w = fmaf(wk[u], h[u].w, acc.w);
        }
      }
    }
    float4 gnow = make_float4(0.f, 0.f, 0.f, 0.f);
    __syncthreads();                                         // the previous task's readers of red / stat are done
    if (sp == 0) {
      // LN of the gate row (C floats): the current position's history row and its own term
      const float* gate = r.u + (long long)b * r.hid + C;
      float s = 0.f;
      for (int c = threadIdx.x * 4; c < C; c += TPB * 4) { const float4 v = __ldcg(reinterpret_cast<const float4*>(gate + c)); s += (v.x + v.y) + (v.z + v.w); }
      const float mean = block_sum(s, stat) / C;
      float qq = 0.f;
      for (int c = threadIdx.x * 4; c < C; c += TPB * 4) {
        const float4 v = __ldcg(reinterpret_cast<const float4*>(gate + c));
        const float a0 = v.x - mean, a1 = v.y - mean, a2 = v.z - mean, a3 = v.w - mean;
        qq += (a0 * a0 + a1 * a1) + (a2 * a2 + a3 * a3);
      }
      const float rstd = rsqrtf(block_sum(qq, stat + WPB) / C + 1e-5f);
      const float4 gv = __ldcg(reinterpret_cast<const float4*>(gate + c0));
      const float4 sc = *reinterpret_cast<const float4*>(L.ln_scale + c0);
      gnow.x = (gv.x - mean) * rstd * sc.x; gnow.y = (gv.y - mean) * rstd * sc.y;
      gnow.z = (gv.z - mean) * rstd * sc.z; gnow.w = (gv.w - mean) * rstd * sc.w;
      if (warp == 0) *reinterpret_cast<float4*>(hist + (long long)pos * C + c0) = gnow;
    }
    *reinterpret_cast<float4*>(red + warp * 128 + lane * 4) = acc;
    __syncthreads();
    if (warp == 0) {
      float4 tot = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
      for (int k = 0; k < WPB; ++k) {
        const float4 v = *reinterpret_cast<const float4*>(red + k * 128 + lane * 4);
        tot.x += v.x; tot.y += v.y; tot.z += v.z; tot.w += v.w;
      }
      if (sp == 0) {
        const float wp = __ldg(wrow + pos), bp = L.b[pos];    // the current position's own term + spatial bias
        tot.x = fmaf(wp, gnow.x, tot.x) + bp; tot.y = fmaf(wp, gnow.y, tot.y) + bp;
        tot.z = fmaf(wp, gnow.z, tot.z) + bp; tot.w = fmaf(wp, gnow.w, tot.w) + bp;
      }
      *reinterpret_cast<float4*>(r.sg + ((long long)sp * r.B + b) * C + c0) = tot;
    }
  }
}

// ------------------------------------------------------------------------------------------------ sampler (one sequence per CTA)
// Block reductions of the samplers: every thread gets the result.  red: [WPB] floats, then [WPB] ints at red + 32; the
// barrier in front lets the caller reuse `red` right after it read the previous result.
static __device__ __forceinline__ float bmax(float m, float* red) {
  m = warp_max(m);
  __syncthreads();
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = m;
  __syncthreads();
  m = red[0];
#pragma unroll
  for (int k = 1; k < WPB; ++k) m = fmaxf(m, red[k]);
  return m;
}
static __device__ __forceinline__ float bsum(float v, float* red) {                 // fixed order: independent of the grid
  v = warp_sum(v);
  __syncthreads();
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  float s = 0.f;
#pragma unroll
  for (int k = 0; k < WPB; ++k) s += red[k];
  return s;
}
// the first maximal index over the CTA of (bv, bi) (ties go to the lower index)
static __device__ __forceinline__ int bargmax(float bv, int bi, float* red) {
  int* redi = reinterpret_cast<int*>(red + 32);
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) {
    const float ov = __shfl_xor_sync(0xffffffffu, bv, off);
    const int oi = __shfl_xor_sync(0xffffffffu, bi, off);
    if (ov > bv || (ov == bv && oi < bi)) { bv = ov; bi = oi; }
  }
  __syncthreads();
  if ((threadIdx.x & 31) == 0) { red[threadIdx.x >> 5] = bv; redi[threadIdx.x >> 5] = bi; }
  __syncthreads();
  float fv = red[0];
  int fi = redi[0];
#pragma unroll
  for (int k = 1; k < WPB; ++k) {
    const float ov = red[k];
    const int oi = redi[k];
    if (ov > fv || (ov == fv && oi < fi)) { fv = ov; fi = oi; }
  }
  return fi;
}
// The k-th largest of sv[0 .. V) with multiplicity, by an O(V^2) rank count over shared memory.  The thread that finds it
// writes red[48].  Where none does (NaN logits), red[48] keeps what the caller put there: sampler 1 seeds it with -inf
// under constraints; otherwise (sampler 0 always) it is whatever the scratch last held, i.e. undefined.
static __device__ __forceinline__ float kth_largest(const float* sv, int V, int k, float* red) {
  for (int c = threadIdx.x; c < V; c += TPB) {
    const float v = sv[c];
    int gt = 0, ge = 0;
#pragma unroll 8
    for (int j = 0; j < V; ++j) { const float u = sv[j]; gt += u > v; ge += u >= v; }
    if (gt < k && k <= ge) red[48] = v;
  }
  __syncthreads();
  return red[48];
}
static __device__ __forceinline__ int clamp_id(int id, int V) { return id < 0 ? 0 : (id >= V ? V - 1 : id); }
// x[b] = the embedding row of token id (clamped into the vocabulary), by the whole CTA
static __device__ __forceinline__ void embed_row(float* x, const float* embed, int b, int id, int V, int d) {
  id = clamp_id(id, V);
  for (int c = threadIdx.x * 4; c < d; c += TPB * 4)
    *reinterpret_cast<float4*>(x + (long long)b * d + c) = *reinterpret_cast<const float4*>(embed + (long long)id * d + c);
}

// utils.py:97-129: top-k filter keeps logits > (k-th largest), the rest become 0.0 and lose their noise; argmax(logits +
// gumbel) (first maximal index); seq[pos + 1] += index (ADD, quirk Q5).  Then the next position's embedding row.
static __device__ void sample_phase(const progen_decode_run_t& r, int pos, float* sv /* smem [V] */, float* red) {
  const int t = threadIdx.x, V = r.V;
  for (int b = blockIdx.x; b < r.B; b += gridDim.x) {
    __syncthreads();
    const float* lg = r.logits + (long long)b * V;
    if (pos + 1 >= r.n) {
      if (r.logits_all) for (int c = t; c < V; c += TPB) r.logits_all[((long long)b * r.n + pos) * V + c] = __ldcg(lg + c);
      continue;                                                                // nothing after the end
    }
    int tok = r.seq[(long long)b * r.n + pos + 1];
    const bool draw = pos + 1 >= r.start[b];                                   // (before its start the prime is kept)
    if (draw || r.logits_all) {
      for (int c = t; c < V; c += TPB) {
        const float v = __ldcg(lg + c);
        sv[c] = v;
        if (r.logits_all) r.logits_all[((long long)b * r.n + pos) * V + c] = v;
      }
    }
    if (draw) {
      __syncthreads();
      const float kth = r.top_k > 0 ? kth_largest(sv, V, r.top_k, red) : -INFINITY;
      // first maximal index of (kept logit + noise | 0.0): thread-strided scan, then the block arg-max
      float bv = -INFINITY;
      int bi = 0x7fffffff;
      for (int c = t; c < V; c += TPB) {
        const float v = sv[c];
        const bool keep = r.top_k > 0 ? v > kth : true;
        const float nz = r.noise ? r.noise[((long long)b * r.n + pos) * V + c] : 0.f;
        const float x = keep ? v + nz : 0.f;
        if (x > bv) { bv = x; bi = c; }                                        // ascending c: keeps the first maximum
      }
      tok += bargmax(bv, bi, red);
      if (t == 0) r.seq[(long long)b * r.n + pos + 1] = tok;
    }
    // the next position's embedding row (its token is final now), so the next step starts at layer 0 without a phase
    embed_row(r.x, r.embed, b, tok, V, r.d);
  }
}

// ------------------------------------------------------------------------------------------------ standard sampler (sampler 1)
// Philox4x32-10 (Salmon et al., SC'11): 10 rounds of the two 32 x 32 -> 64 multiplications, key bumped between rounds
static __device__ __forceinline__ uint4 philox4x32_10(uint4 c, uint32_t k0, uint32_t k1) {
#pragma unroll
  for (int i = 0; i < 10; ++i) {
    if (i > 0) { k0 += 0x9E3779B9u; k1 += 0xBB67AE85u; }
    const uint32_t lo0 = 0xD2511F53u * c.x, hi0 = __umulhi(0xD2511F53u, c.x);
    const uint32_t lo1 = 0xCD9E8D57u * c.z, hi1 = __umulhi(0xCD9E8D57u, c.z);
    c = make_uint4(hi1 ^ c.y ^ k0, lo1, hi0 ^ c.w ^ k1, lo0);
  }
  return c;
}
// Gumbel noise of token c at position p of the stream `sid` (the layout is spelled out in progen_b200.h; tests replay it)
static __device__ __forceinline__ float philox_gumbel(unsigned long long seed, long long sid, int p, int c) {
  const uint4 o = philox4x32_10(make_uint4((uint32_t)c >> 2, (uint32_t)p, (uint32_t)sid, (uint32_t)((unsigned long long)sid >> 32)),
                                (uint32_t)seed, (uint32_t)(seed >> 32));
  const uint32_t x = (c & 3) == 0 ? o.x : ((c & 3) == 1 ? o.y : ((c & 3) == 2 ? o.z : o.w));
  const float u = (float)(2u * (x >> 9) + 1u) * 5.9604644775390625e-8f;        // (2 (x >> 9) + 1) 2^-24: exact, in (0, 1)
  return -logf(-logf(u));
}

// Sampler 1 (one sequence per CTA, like sample_phase): top-k (ties at the k-th largest kept) -> softmax(l / T) -> nucleus
// (smallest q-descending prefix reaching top_p) -> first maximal l / T + Gumbel over the kept ids; T == 0: first maximal raw
// logit.  seq[p+1] = id (a write), token_logp = l[id] - logsumexp(l) (the unfiltered model at T = 1), id 0 ends the
// sequence (end[b], one atomicAdd on n_ended).  Not inlined, and only reached through the uniform `sampler` branch, so its
// registers stay out of the GEMV phases' allocation.  sv: shared memory [2 V]; red: the block-reduction scratch.
// Constraints (progen_b200.h): after logsumexp of the raw logits, sv is overwritten with the adjusted logits a, and the
// filter and draw below run on a unchanged: -inf and NaN never win a comparison, so only candidates can be drawn.
// One argument (fewer registers at the call): the logit bias, the repetition penalty, min_new_tokens, the position
// tables (pbias [tables, plen, V], ptable [rows]: each row's table or -1; pbias null = none) and the motif descriptor
// (null = none) with the launch's max_length, which its lookahead counts the positions left against
struct SampleCons {
  const float* bias; float theta; int window, min_new; const float* pbias; const int32_t* ptable; int plen;
  const progen_motif_t* motif; int max_length;
};

// Motif step (progen_b200.h): may id c be drawn by a row in state st ([P] bitsets, flags), given that it is the row's
// first generated token (`first`) and `left` positions follow it before max_length?  With nx, the row's next state after
// c is written there (the caller's c was drawn, so every pattern runs).  At most P <= 9 patterns of 64-bit operations;
// the closure loop runs once per optional position in a row plus one.
static __device__ __forceinline__ uint64_t ldg64(const uint64_t* p) { return __ldg(reinterpret_cast<const unsigned long long*>(p)); }
static __device__ __forceinline__ uint64_t ldcg64(const uint64_t* p) { return __ldcg(reinterpret_cast<const unsigned long long*>(p)); }
static __device__ __forceinline__ bool motif_allows(const progen_motif_t* M, const uint64_t* st, int c, int V, bool first,
                                                    int left, uint64_t* nx) {
  const int P = __ldg(&M->num_patterns);
  const bool req = __ldg(&M->required) != 0;
  const uint64_t flags = ldcg64(st + P);
  if (c == 0) {                                                                // EOS: the row ends after t_L
    if (req && !(flags & 1ull)) return false;
    for (int k = req ? 1 : 0; k < P; ++k) {
      const progen_motif_pattern_t* pt = M->pattern + k;
      if ((ldg64(&pt->anchors) & 2ull) && (ldcg64(st + k) & ldg64(&pt->last))) return false;
    }
    return true;
  }
  bool ok = true;
  uint64_t met = 0;
  for (int k = 0; k < P; ++k) {
    const progen_motif_pattern_t* pt = M->pattern + k;
    const uint64_t anch = ldg64(&pt->anchors), opt = ldg64(&pt->optional), last = ldg64(&pt->last);
    const bool z = !(anch & 1ull) || first;                                    // the start state is active at c
    const uint64_t D = ldcg64(st + k) | (z ? ldg64(&pt->lead) : 0ull);
    uint64_t X = ((D << 1) | (z ? 1ull : 0ull)) & ldg64(M->mask + (long long)k * V + c);
    for (uint64_t Y = X | ((X << 1) & opt); Y != X; Y = X | ((X << 1) & opt)) X = Y;
    const bool hit = (X & last) != 0ull;
    if (k == 0 && req) {
      met = ((anch & 2ull) ? 0ull : (flags & 1ull)) | (hit ? 1ull : 0ull);
      if (!met) {
        // need[] never increases along the pattern: the state's fewest residues left are those of its highest bit
        const int need = X ? __ldg(&M->need[63 - __clzll((long long)X)]) : (!(anch & 1ull) ? __ldg(&M->need[64]) : 0x7fffffff);
        if (need > left) ok = false;
      }
    } else if (hit && (!(anch & 2ull) || left == 0)) {
      ok = false;
    }
    if (nx) nx[k] = X;
    else if (!ok) return false;
  }
  if (nx) nx[P] = met;
  return ok;
}
// The queue kernels' view of the slots (SLOT): this step's row and position of every slot (shared memory), the queue's
// device state and what a refill resets.  Without a queue (slot_row null) srow[b] = b and spos[b] = the launch's position.
struct SlotArgs {
  const int* srow; const int* spos;
  int32_t* slot_row; int32_t* slot_pos; int32_t* next_row; int32_t* done;
  const progen_decode_layer_t* layers;
  int depth, num_rows, max_length, shift_tokens;
};
static __device__ __forceinline__ SlotArgs slot_args() { return SlotArgs{}; }
static __device__ __forceinline__ SlotArgs slot_args(const SlotArgs& s) { return s; }
// SLOT: the queue kernels pass one SlotArgs (`slot`); the single-stream kernels pass none, so their call is unchanged
template <bool SLOT, typename... SA>
static __device__ __noinline__ void sample_std_phase(const float* logits, int32_t* seq, const int32_t* start, int32_t* end, int32_t* n_ended,
                                                     float* token_logp, float* logits_all, const float* embed, float* x,
                                                     const int64_t* sample_id, int n, int V, int d, int B, int top_k, float temp,
                                                     float top_p, unsigned long long seed, SampleCons cs, int pos_, float* sv, float* red,
                                                     SA... slot) {
  static_assert(TPB >= 256, "V <= 512: at most two ids per thread");
  static_assert(sizeof...(SA) == (SLOT ? 1 : 0), "one SlotArgs with SLOT");
  const int t = threadIdx.x;
  float* qv = sv + V;                                                          // kept ids: q; removed: -1
  int* redi = reinterpret_cast<int*>(red + 32);
  const bool cons = cs.bias != nullptr || cs.theta != 1.f || cs.min_new != 0 || cs.pbias != nullptr || cs.motif != nullptr;  // uniform
  const SlotArgs S = slot_args(slot...);
  // queue: slot b retires its row (counted in `done`), then claims the next row of the queue, q = next_row++.  A claimed
  // row starts at position 0: the slot's token-shift slot 0 of every layer (the only state read at position 0 before it
  // is written) is zeroed and x takes the embedding of the row's BOS.  With no row left the slot goes idle.
  auto refill = [&](int b) {
    __syncthreads();                                                           // the draw's readers of red / redi are done
    if (t == 0) { atomicAdd(S.done, 1); redi[0] = atomicAdd(S.next_row, 1); }
    __syncthreads();
    const int q = redi[0];
    const bool got = q < S.num_rows;
    if (t == 0) { S.slot_row[b] = got ? q : -1; S.slot_pos[b] = 0; }
    if (got && S.shift_tokens) {
      for (int li = 0; li < S.depth; ++li) {
        float* s1 = S.layers[li].shift1 + (long long)b * d;                    // [B][2][d/2]: slot 0 of row b
        float* s2 = S.layers[li].shift2 + (long long)b * d;
        for (int c = t; c < (d >> 1); c += TPB) { s1[c] = 0.f; s2[c] = 0.f; }
      }
    }
    const int id = clamp_id(got ? seq[(long long)q * n] : 0, V);
    for (int c = t * 4; c < d; c += TPB * 4)
      *reinterpret_cast<float4*>(x + (long long)b * d + c) = *reinterpret_cast<const float4*>(embed + (long long)id * d + c);
  };
  for (int b = blockIdx.x; b < B; b += gridDim.x) {
    __syncthreads();
    const float* lg = logits + (long long)b * V;
    int rb = b, pos = pos_;                                                    // the row slot b decodes, and its position
    if constexpr (SLOT) {
      rb = S.srow[b]; pos = S.spos[b];
      if (rb < 0) {                                                            // idle: only the slot's own scratch (x stays finite)
        for (int c = t * 4; c < d; c += TPB * 4)
          *reinterpret_cast<float4*>(x + (long long)b * d + c) = *reinterpret_cast<const float4*>(embed + c);
        continue;
      }
    }
    const long long row = (long long)rb * n;
    if (pos + 1 >= n) {
      if (logits_all) for (int c = t; c < V; c += TPB) logits_all[(row + pos) * V + c] = __ldcg(lg + c);
      if constexpr (SLOT) { if (S.slot_row) refill(b); }
      continue;
    }
    int tok = seq[row + pos + 1];
    const bool draw = pos + 1 >= start[rb] && pos + 1 < end[rb];               // (after its EOS a sequence stays 0)
    if (draw || logits_all) {
      for (int c = t; c < V; c += TPB) {
        const float v = __ldcg(lg + c);
        sv[c] = v;
        if (logits_all) logits_all[(row + pos) * V + c] = v;
      }
    }
    if (draw) {
      __syncthreads();
      float m = -INFINITY;
      for (int c = t; c < V; c += TPB) m = fmaxf(m, sv[c]);
      m = bmax(m, red);
      float s = 0.f;
      for (int c = t; c < V; c += TPB) s += expf(sv[c] - m);
      const float lse = m + logf(bsum(s, red));
      if (cons) {
        // presence flags of the ids at positions max(1, p + 1 - W) .. p, in the q half (filled only after this)
        int* seen = reinterpret_cast<int*>(qv);
        const bool pen = cs.theta != 1.f;
        if (pen) {
          for (int c = t; c < V; c += TPB) seen[c] = 0;
          __syncthreads();
          for (int j = (cs.window > 0 ? max(1, pos + 1 - cs.window) : 1) + t; j <= pos; j += TPB) {
            const int c = __ldcg(seq + row + j);
            if (c >= 0 && c < V) seen[c] = 1;
          }
          __syncthreads();
        }
        const bool no_eos = pos + 1 < start[rb] + cs.min_new;
        const float* pb = nullptr;                                              // the row's table row at offset j
        if (cs.pbias) {
          const int tb = __ldg(cs.ptable + rb), j = pos + 1 - start[rb];       // (j >= 0: a drawn position)
          if (tb >= 0 && j < cs.plen) pb = cs.pbias + ((long long)tb * cs.plen + j) * V;
        }
        const uint64_t* mst = nullptr;                                          // the row's motif state
        if (cs.motif) mst = cs.motif->state + (long long)rb * (cs.motif->num_patterns + 1);
        float ma = -INFINITY;
        for (int c = t; c < V; c += TPB) {
          float a = sv[c];
          if (pen && seen[c]) a = a > 0.f ? __fdiv_rn(a, cs.theta) : __fmul_rn(a, cs.theta);
          if (cs.bias) a = __fadd_rn(a, __ldg(cs.bias + c));                 // (no FMA with the penalty's product)
          if (pb) a = __fadd_rn(a, __ldg(pb + c));                            // a separate rounding after the bias
          if (c == 0 && no_eos) a = -INFINITY;
          if (mst && a > -INFINITY && !motif_allows(cs.motif, mst, c, V, pos + 1 == start[rb], cs.max_length - pos - 2, nullptr))
            a = -INFINITY;
          sv[c] = a;
          ma = fmaxf(ma, a);
        }
        if (t == 0) red[48] = -INFINITY;                                        // top-k over fewer candidates than k: keep all
        m = bmax(ma, red);                                                      // the candidates' maximum (NaN skipped)
      }
      int id;
      // a temperature so small that max / T overflows (e.g. 1e-39, subnormal) is the T -> 0 limit: the greedy draw
      if (temp == 0.f || isinf(m / temp)) {
        float bv = -INFINITY;
        int bi = 0x7fffffff;
        for (int c = t; c < V; c += TPB) if (sv[c] > bv) { bv = sv[c]; bi = c; }
        id = bargmax(bv, bi, red);
      } else {
        const float kth = top_k > 0 && top_k < V ? kth_largest(sv, V, top_k, red) : -INFINITY;
        const float mt = m / temp;                                              // the row maximum is always kept
        float z = 0.f;
        for (int c = t; c < V; c += TPB) if (sv[c] >= kth) z += expf(sv[c] / temp - mt);
        z = bsum(z, red);
        for (int c = t; c < V; c += TPB) qv[c] = sv[c] >= kth ? expf(sv[c] / temp - mt) / z : -1.f;
        __syncthreads();
        if (top_p < 1.f) {
          // q-descending order = logit-descending order, ties by lower id; keep c iff the mass strictly before it < top_p
          bool drop[2] = {false, false};
#pragma unroll
          for (int i = 0; i < 2; ++i) {
            const int c = t + i * TPB;
            if (c < V && qv[c] >= 0.f) {
              const float v = sv[c];
              float before = 0.f;
              for (int j = 0; j < V; ++j) {
                const float u = sv[j], qj = qv[j];
                if (qj >= 0.f && (u > v || (u == v && j < c))) before += qj;
              }
              drop[i] = !(before < top_p);
            }
          }
          __syncthreads();
#pragma unroll
          for (int i = 0; i < 2; ++i) if (drop[i]) qv[t + i * TPB] = -1.f;
          __syncthreads();
        }
        float bv = -INFINITY;
        int bi = 0x7fffffff;
        const long long sid = sample_id[rb];
        for (int c = t; c < V; c += TPB) {
          if (qv[c] < 0.f) continue;
          const float sc = sv[c] / temp + philox_gumbel(seed, sid, pos + 1, c);
          if (sc > bv) { bv = sc; bi = c; }
        }
        id = bargmax(bv, bi, red);
      }
      if (id >= V) id = 0;                                                      // no candidate compared (NaN logits): EOS
      tok = id;
      if (t == 0) {
        seq[row + pos + 1] = id;
        if (token_logp) token_logp[row + pos + 1] = (cons ? __ldcg(lg + id) : sv[id]) - lse;   // the raw logit
        if (id == 0) { end[rb] = pos + 1; atomicAdd(n_ended, 1); }
        else if (cons && cs.motif) {                                           // the drawn residue's next state (read next draw, after the grid barrier)
          uint64_t* mst = cs.motif->state + (long long)rb * (cs.motif->num_patterns + 1);
          motif_allows(cs.motif, mst, id, V, pos + 1 == start[rb], cs.max_length - pos - 2, mst);
        }
      }
    }
    if constexpr (SLOT) {
      if (S.slot_row) {                                                        // retire at EOS or at the last position
        if ((draw && tok == 0) || pos + 1 >= S.max_length - 1) { refill(b); continue; }
        if (t == 0) S.slot_pos[b] = pos + 1;
      }
    }
    const int id = clamp_id(tok, V);
    for (int c = t * 4; c < d; c += TPB * 4)
      *reinterpret_cast<float4*>(x + (long long)b * d + c) = *reinterpret_cast<const float4*>(embed + (long long)id * d + c);
  }
}

enum { K_NONE = 0, K_GEMV = 1, K_ATT = 2, K_SGU = 3, K_SAMPLE = 4 };
struct PhaseEnt { int kind, next; Phase ph; };     // next: table index of the following GEMV phase (weights to prefetch)
static __host__ __device__ int num_phases(int depth) { return depth * 7 + 2; }

// Phase table (shared memory, built once per launch): per layer QKV | attention | out-proj | FF-in | [SGU | SGU proj] | FF-out,
// then final LN + head, sampler.  Position-dependent fields (pos) are filled in at use.
static __device__ void build_phase_table(const progen_decode_run_t& r, PhaseEnt* tab, bool att_consumer_merge, int nsplit) {
  const int d = r.d, I = r.inner, hid = r.hid;
  const int nph = num_phases(r.depth);
  for (int li = threadIdx.x; li < r.depth; li += TPB) {
    const progen_decode_layer_t L = r.layers[li];
    PhaseEnt* e = tab + li * 7;
    for (int j = 0; j < 7; ++j) { e[j].kind = K_NONE; e[j].next = 0; e[j].ph = Phase{}; }
    Phase ph{};
    // LN + shift + QKV + rotary + cache
    ph.wt = L.wqkv_t; ph.bias = nullptr; ph.xin = r.x; ph.ldx = d; ph.out = r.q; ph.ldo = I; ph.N = 3 * I; ph.K = d; ph.epi = EP_ROTARY_CACHE;
    ph.pro = PRO_LN; ph.ln_scale = L.ln1_scale; ph.ln_prev = r.shift_tokens ? L.shift1 : nullptr;
    ph.kcache = L.kcache; ph.vcache = L.vcache; ph.inner = I; ph.dim_head = r.dim_head; ph.n = r.n; ph.rot_sin = r.rot_sin; ph.rot_cos = r.rot_cos;
    ph.g = make_geo(ph);
    e[0].kind = K_GEMV; e[0].ph = ph; e[0].next = li * 7 + 2;
    ph = Phase{}; ph.kcache = L.kcache; ph.vcache = L.vcache;
    e[1].kind = K_ATT; e[1].ph = ph;
    // out-proj + residual
    ph = Phase{};
    ph.wt = L.wo_t; ph.bias = L.bo; ph.xin = r.att; ph.ldx = I; ph.out = r.x; ph.ldo = d; ph.N = d; ph.K = I; ph.epi = EP_RESIDUAL;
    if (att_consumer_merge) { ph.pro = PRO_ATT; ph.aux = r.att_part; ph.window = r.window; ph.dim_head = r.dim_head; }
    ph.g = make_geo(ph);
    e[2].kind = K_GEMV; e[2].ph = ph; e[2].next = li * 7 + 3;
    // LN + shift + FF-in (+ GLU / GELU)
    ph = Phase{};
    ph.wt = L.win_t; ph.bias = L.bin; ph.xin = r.x; ph.ldx = d; ph.out = r.u; ph.ldo = hid; ph.N = hid; ph.K = d;
    ph.epi = L.kind == 0 ? EP_GLU : EP_GELU; ph.pro = PRO_LN; ph.ln_scale = L.ln2_scale; ph.ln_prev = r.shift_tokens ? L.shift2 : nullptr;
    ph.g = make_geo(ph);
    e[3].kind = K_GEMV; e[3].ph = ph; e[3].next = li * 7 + (L.kind == 2 ? 5 : 6);
    const float* last = r.u;
    int last_k = hid;
    if (L.kind == 2) {
      ph = Phase{}; ph.ln_scale = L.sgu_ln_scale; ph.wt = L.sgu_w; ph.bias = L.sgu_b; ph.kcache = L.gn_hist;
      e[4].kind = K_SGU; e[4].ph = ph;
      ph = Phase{};
      ph.wt = L.sgu_proj_t; ph.bias = L.sgu_proj_b; ph.xin = r.u; ph.ldx = hid; ph.out = r.pj; ph.ldo = hid / 2; ph.N = hid / 2; ph.K = hid / 2;
      ph.epi = EP_BIAS; ph.pro = PRO_SGU; ph.aux = r.sg; ph.nsplit = nsplit; ph.aux_stride = (long long)r.B * (hid / 2);
      ph.g = make_geo(ph);
      e[5].kind = K_GEMV; e[5].ph = ph; e[5].next = li * 7 + 6;
      last = r.pj; last_k = hid / 2;
    }
    // FF-out + residual
    ph = Phase{};
    ph.wt = L.wout_t; ph.bias = L.bout; ph.xin = last; ph.ldx = last_k; ph.out = r.x; ph.ldo = d; ph.N = d; ph.K = last_k; ph.epi = EP_RESIDUAL;
    ph.g = make_geo(ph);
    e[6].kind = K_GEMV; e[6].ph = ph; e[6].next = li + 1 < r.depth ? (li + 1) * 7 : nph - 2;
  }
  if (threadIdx.x == 0) {
    // final LN + logits (progen.py:219-222), then the sampler
    Phase ph{};
    ph.wt = r.whead_t; ph.bias = r.bhead; ph.xin = r.x; ph.ldx = d; ph.out = r.logits; ph.ldo = r.V; ph.N = r.V; ph.K = d; ph.epi = EP_BIAS;
    ph.pro = PRO_LN; ph.ln_scale = r.lnf_scale; ph.ln_prev = nullptr;
    ph.g = make_geo(ph);
    tab[nph - 2].kind = K_GEMV; tab[nph - 2].ph = ph; tab[nph - 2].next = 0;
    tab[nph - 1].kind = K_SAMPLE; tab[nph - 1].next = 0; tab[nph - 1].ph = Phase{};
  }
  __syncthreads();
}

static constexpr size_t MAX_SMEM = 227 * 1024;
template <int BT, bool TCW> static constexpr size_t decode_smem_floats() {
  using TL = Tile<BT, TCW>;
  return (size_t)BT * TL::XP + TL::PART + TL::STATF + TL::WSM + WPB * 128 + 64;
}
// dynamic shared memory of a launch: the tile regions, the phase table and (single stream, when they fit) the unit tables
template <int BT, bool TCW> static __host__ __device__ size_t decode_smem_bytes(int depth, bool with_unit_tables) {
  return decode_smem_floats<BT, TCW>() * sizeof(float) + (size_t)num_phases(depth) * (sizeof(PhaseEnt) + (with_unit_tables ? WSEGS * (sizeof(UnitEnt) + sizeof(FinEnt)) : 0)) + 16;
}

// STD: sampler 1 (a separate instantiation, so the sampler-0 kernels compile exactly as they do without it)
template <int BT, typename TW, bool STD>
static __device__ __forceinline__ void run(const progen_decode_run_t& r) {
  extern __shared__ __align__(16) float smem[];
  using TL = Tile<BT, sizeof(TW) == 2>;
  float* xs = smem;                                    // [BT][XP]
  float* part = xs + BT * TL::XP;                      // partial sums
  float* stat = part + TL::PART;                       // [STATF]
  float* wsm = stat + TL::STATF;                       // B > 8: one wave's weights
  float* red = wsm + TL::WSM;                          // scratch of the other phases: WPB * 128 + 64
  PhaseEnt* tab = reinterpret_cast<PhaseEnt*>(red + WPB * 128 + 64);
  __shared__ __align__(8) uint64_t stage_bar;
  const uint32_t sbar = smem_u32(&stage_bar);
  uint32_t sparity = 0;
  if (threadIdx.x == 0) { mbar_init(sbar, 1); fence_barrier_init(); }
  const int nph = num_phases(r.depth);
  constexpr bool MERGE_IN_ATT = BT > 1;
  const bool att_consumer = !MERGE_IN_ATT && r.inner <= 4 * TPB;
  // The attention's warps per (sequence, head) and the SGU's split of the history range follow the number of sequences
  // they are planned for.  Sampler 0 plans for the B of the launch.  Sampler 1 plans for the most sequences of the batch
  // tile's class (1, 2-8, 9-64), so a row's arithmetic does not depend on how many rows share its launch.
  constexpr int PLAN = STD ? (BT == 1 ? 1 : (BT <= 8 ? 8 : 64)) : 0;
  build_phase_table(r, tab, att_consumer, sgu_splits<PLAN>(r));
  const bool use_tabs = BT == 1 && decode_smem_bytes<BT, sizeof(TW) == 2>(r.depth, true) <= MAX_SMEM;
  UnitEnt* utab = reinterpret_cast<UnitEnt*>((reinterpret_cast<uintptr_t>(tab + nph) + 15) & ~(uintptr_t)15);   // [nph][WSEGS]   (single stream only)
  FinEnt* ftab = reinterpret_cast<FinEnt*>(utab + (use_tabs ? nph * WSEGS : 0));
  if (use_tabs) {
    for (int idx = threadIdx.x; idx < nph * WSEGS; idx += TPB) {
      const int e = idx / WSEGS, u = idx % WSEGS;
      if (tab[e].kind == K_GEMV) build_unit_tables(tab[e].ph, utab + e * WSEGS, ftab + e * WSEGS, u);
    }
    __syncthreads();
  }
  for (int i = threadIdx.x; i < BT * TL::XP; i += TPB) xs[i] = 0.f;     // tails beyond K are multiplied by zero weights: keep them finite
  __syncthreads();
  unsigned int round = 0;
  const int d = r.d, B = r.B;
  Prof pf{r.prof, 0, false};
  WRegs<TW> w;
  Pre pre{};
  bool have = false;                                   // `w`, `pre` hold the next GEMV phase's prefetch
  // The queue kernels (sampler 1, B > 1) keep a row and a position per slot (DESIGN.md §3.3): every phase reads
  // slot b's position from s_pos[b], copied at the top of each step from slot_pos (which the sampler phase advances), or
  // the launch's position for every slot when the launch has no queue.
  constexpr bool SLOT = STD && BT > 1;
  const bool queue = SLOT && r.slot_row != nullptr;
  int* s_row = nullptr;
  int* s_pos = nullptr;
  if constexpr (SLOT) {
    __shared__ int slot_sh[2 * 64];
    s_row = slot_sh;
    s_pos = slot_sh + 64;
  }
  for (int step = 0; step < r.nsteps; ++step) {
    const int pos = r.pos0 + step;
    pf.on = r.prof != nullptr && step == r.nsteps - 1 && (blockIdx.x == 0 || blockIdx.x == gridDim.x - 1);
    pf.ev = 0;
    if constexpr (SLOT) {
      if (threadIdx.x < B) {
        s_row[threadIdx.x] = queue ? __ldcg(r.slot_row + threadIdx.x) : (int)threadIdx.x;
        s_pos[threadIdx.x] = queue ? __ldcg(r.slot_pos + threadIdx.x) : pos;
      }
      __syncthreads();
    }
    if (step == 0) {
      // embedding of the launch's first position (later ones are written by the sampler phase)
      for (int idx = blockIdx.x * TPB + threadIdx.x; idx < B * (d >> 2); idx += gridDim.x * TPB) {
        const int b = idx / (d >> 2), c = (idx % (d >> 2)) * 4;
        int id;
        if constexpr (SLOT) id = s_row[b] < 0 ? 0 : r.seq[(long long)s_row[b] * r.n + s_pos[b]];
        else id = r.seq[(long long)b * r.n + pos];
        id = clamp_id(id, r.V);
        *reinterpret_cast<float4*>(r.x + (long long)b * d + c) = *reinterpret_cast<const float4*>(r.embed + (long long)id * d + c);
      }
      grid_sync(r.grid_bar, round, pf);
    }
    for (int e = 0; e < nph; ++e) {
      const int kind = tab[e].kind;
      if (kind == K_NONE) continue;
      bool fetch_next = false;
      if (kind == K_GEMV) {
        Phase ph = tab[e].ph;
        ph.pos = pos;
        if (!have) prefetch_phase<BT, TW>(ph, w, pre, use_tabs ? utab + e * WSEGS : nullptr, use_tabs ? ftab + e * WSEGS : nullptr);
        prof_mark(pf, 0);
        if (B <= BT) {
          gemv_phase<BT, TW, SLOT>(ph, B, xs, part, stat, wsm, w, pre, pf, sbar, sparity, false, s_pos);
        } else {
          // more sequences than the batch tile: sub-batches of BT sequences run through the phase one after the other with
          // the same weights (per warp, 32 sequences cost 4 LayerNorm rows and 8 k-steps; a 64-wide tile costs twice that
          // in series, and half the shared memory of a 64-wide tile)
          for (int b0 = 0; b0 < B; b0 += BT) {
            if (b0 > 0) __syncthreads();                       // every warp is done reading the previous pass's staged rows
            Phase ps = ph;
            if (ps.xin) ps.xin += (long long)b0 * ps.ldx;
            ps.out += (long long)b0 * ps.ldo;
            if (ps.ln_prev) ps.ln_prev += (long long)b0 * ps.K;
            if (ps.kcache) { ps.kcache += (long long)b0 * ps.n * ps.inner; ps.vcache += (long long)b0 * ps.n * ps.inner; }
            if (ps.pro == PRO_SGU) ps.aux += (long long)b0 * ps.K;
            gemv_phase<BT, TW, SLOT>(ps, min(BT, B - b0), xs, part, stat, wsm, w, pre, pf, sbar, sparity, b0 > 0, SLOT ? s_pos + b0 : nullptr);
          }
        }
        prof_mark(pf, 3);
        have = fetch_next = !(e == nph - 2 && step + 1 == r.nsteps);
      } else if (kind == K_ATT) {
        if (MERGE_IN_ATT || !att_consumer) {
          attention_batch<PLAN, SLOT>(r, tab[e].ph.kcache, tab[e].ph.vcache, pos, red, s_pos);
        } else {
          attention_phase(r, tab[e].ph.kcache, tab[e].ph.vcache, pos, red);
        }
      } else if (kind == K_SGU) {
        const SguArgs sa{tab[e].ph.ln_scale, reinterpret_cast<const float*>(tab[e].ph.wt), tab[e].ph.bias, tab[e].ph.kcache};
        sgu_phase<PLAN, SLOT>(r, sa, pos, red, s_pos);
      } else if constexpr (SLOT) {
        sample_std_phase<true>(r.logits, r.seq, r.start, r.end, r.n_ended, r.token_logp, r.logits_all, r.embed, r.x, r.sample_id, r.n, r.V,
                               d, B, r.top_k, r.temperature, r.top_p, r.seed,
                               SampleCons{r.logit_bias, r.repetition_penalty, r.repetition_window, r.min_new_tokens, r.position_bias,
                                          r.position_bias_table, r.position_bias_len, r.motif, r.max_length}, pos, xs, red,
                               SlotArgs{s_row, s_pos, r.slot_row, r.slot_pos, r.next_row, r.done, r.layers, r.depth, r.num_rows,
                                        r.max_length, r.shift_tokens});
      } else if constexpr (STD) {
        sample_std_phase<false>(r.logits, r.seq, r.start, r.end, r.n_ended, r.token_logp, r.logits_all, r.embed, r.x, r.sample_id, r.n, r.V,
                                d, B, r.top_k, r.temperature, r.top_p, r.seed,
                                SampleCons{r.logit_bias, r.repetition_penalty, r.repetition_window, r.min_new_tokens, r.position_bias,
                                          r.position_bias_table, r.position_bias_len, r.motif, r.max_length}, pos, xs, red);
      } else {
        sample_phase(r, pos, xs, red);
      }
      // arrive, THEN fetch the next GEMV phase's weights and operands (nothing of it depends on other CTAs' output of
      // this phase), then wait: the instructions and the loads overlap the barrier's latency
      long long t0 = 0;
      grid_arrive(r.grid_bar, round, pf, t0);
      if (fetch_next) {
        Phase nx = tab[tab[e].next].ph;
        nx.pos = e == nph - 2 ? pos + 1 : pos;               // the head's successor is layer 0 of the next position
        prefetch_phase<BT, TW>(nx, w, pre, use_tabs ? utab + tab[e].next * WSEGS : nullptr, use_tabs ? ftab + tab[e].next * WSEGS : nullptr);
        prof_mark(pf, 4);
      }
      grid_wait(r.grid_bar, round, pf, t0);
      if (STD && kind == K_SAMPLE) {
        // EOS early exit: the barrier above orders every CTA's count of this sampler phase before the read, and nothing
        // writes the counter before the next sampler phase, so every CTA sees the same value and leaves together.  With a
        // queue the count is of retired rows (EOS or the last position), and the launch ends when all Q have retired.
        const int32_t* cnt = r.n_ended;
        int goal = B;
        if constexpr (SLOT) {
          if (queue) { cnt = r.done; goal = r.num_rows; }
        }
        int ended;
        asm volatile("ld.acquire.gpu.global.s32 %0, [%1];" : "=r"(ended) : "l"(cnt) : "memory");
        if (ended >= goal) {
          if (blockIdx.x == 0 && threadIdx.x == 0) *r.steps_run = step + 1;
          return;
        }
      }
    }
  }
  if (STD && blockIdx.x == 0 && threadIdx.x == 0) *r.steps_run = r.nsteps;
}

template <int BT, typename TW, bool STD>
__global__ void __launch_bounds__(TPB, 1) decode_persistent_kernel(const progen_decode_run_t r) {
  run<BT, TW, STD>(r);
}

template <int BT, typename TW, bool STD>
int launch_run_sampler(const progen_decode_run_t& r, cudaStream_t s) {
  using TL = Tile<BT, sizeof(TW) == 2>;
  static_assert((BT * TL::XP) % 4 == 0 && TL::PART % 4 == 0 && TL::WSM % 4 == 0, "the scratch regions must stay 16-byte aligned");
  size_t smem = decode_smem_bytes<BT, sizeof(TW) == 2>(r.depth, BT == 1);
  if (smem > MAX_SMEM) smem = decode_smem_bytes<BT, sizeof(TW) == 2>(r.depth, false);   // deep model: no unit tables
  PG_CHECK_ARG(smem <= MAX_SMEM);                                  // (the phase table itself: depth * 7 + 2 entries)
  if (STD && BT > 1) PG_CHECK_ARG(smem + 2 * 64 * sizeof(int) <= MAX_SMEM);   // + the queue kernels' slot table (static)
  auto kern = decode_persistent_kernel<BT, TW, STD>;
  static size_t set_for = 0;
  if (set_for < smem) {
    PG_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    set_for = smem;
  }
  int per_sm = 0;
  PG_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kern, TPB, smem));
  PG_CHECK_ARG(per_sm >= 1);
  const int grid = pg_num_sms();
  void* args[] = {(void*)&r};
  PG_CUDA(cudaLaunchCooperativeKernel((void*)kern, dim3(grid), dim3(TPB), args, smem, s));
  __atomic_fetch_add(&g_progen_launches, 1ull, __ATOMIC_RELAXED);
  return PROGEN_OK;
}
template <int BT, typename TW>
int launch_run(const progen_decode_run_t& r, cudaStream_t s) {
  return r.sampler == 1 ? launch_run_sampler<BT, TW, true>(r, s) : launch_run_sampler<BT, TW, false>(r, s);
}

}  // namespace

extern "C" {

// Consume positions pos0 .. pos0 + nsteps - 1 of all B sequences in ONE kernel.  `grid_bar` must be zero on entry (the caller
// re-zeroes it before the next launch).
int progen_decode_run(const progen_decode_run_t* r, void* stream) {
  PG_CHECK_ARG(r != nullptr && r->layers != nullptr && r->depth > 0 && r->B >= 1 && r->B <= 64 && r->nsteps >= 0);
  PG_CHECK_ARG(r->d % 8 == 0 && r->inner % 8 == 0 && r->hid % 256 == 0 && r->V % 2 == 0 && r->V <= 512);
  PG_CHECK_ARG(r->d <= 8192 && r->inner <= 8192 && r->hid <= 8192);   // K segments of one pair fit a wave (KS <= WSEGS)
  PG_CHECK_ARG(r->dim_head >= 8 && r->dim_head <= 64 && (r->dim_head & (r->dim_head - 1)) == 0);   // float4 lanes per value row
  PG_CHECK_ARG(r->window >= 1 && r->window <= 512);                    // <= 32 key slices per (sequence, head)
  // row queue: every field or none; sampler 1 on a batched tile only; at least one row per slot
  const bool queue = r->slot_row != nullptr || r->slot_pos != nullptr || r->next_row != nullptr || r->done != nullptr ||
                     r->num_rows != 0;
  PG_CHECK_ARG(r->max_length == 0 || (r->max_length >= 2 && r->max_length <= r->n));
  if (queue) {
    PG_CHECK_ARG(r->sampler == 1 && r->B >= 2 && r->num_rows >= r->B && r->max_length >= 2);
    PG_CHECK_ARG(r->slot_row != nullptr && r->slot_pos != nullptr && r->next_row != nullptr && r->done != nullptr);
    PG_CHECK_ARG(r->logits_all == nullptr || r->num_rows == r->B);
  }
  PG_CHECK_ARG(r->pos0 >= 0 && (queue || r->pos0 + r->nsteps <= r->n));
  PG_CHECK_ARG(r->grid_bar != nullptr && r->att_count != nullptr && r->att_part != nullptr);
  PG_CHECK_ARG(r->sampler == 0 || r->sampler == 1);
  PG_CHECK_ARG(std::isfinite(r->repetition_penalty) && r->repetition_penalty > 0.f);
  PG_CHECK_ARG(r->repetition_window >= 0 && r->repetition_window <= r->n && r->min_new_tokens >= 0 && r->min_new_tokens <= r->n);
  if (r->sampler == 0) PG_CHECK_ARG(r->logit_bias == nullptr && r->repetition_penalty == 1.f && r->min_new_tokens == 0);
  // position tables: both pointers or neither, a length in [1, n], sampler 1 only
  PG_CHECK_ARG((r->position_bias == nullptr) == (r->position_bias_table == nullptr));
  if (r->position_bias) PG_CHECK_ARG(r->sampler == 1 && r->position_bias_len >= 1 && r->position_bias_len <= r->n);
  // motif constraints: sampler 1 with a max_length; the descriptor is device memory, so its header is read back here
  if (r->motif) {
    PG_CHECK_ARG(r->sampler == 1 && r->max_length >= 2);
    progen_motif_t h;
    PG_CUDA(cudaMemcpyAsync(&h, r->motif, sizeof(h), cudaMemcpyDeviceToHost, (cudaStream_t)stream));
    PG_CUDA(cudaStreamSynchronize((cudaStream_t)stream));
    PG_CHECK_ARG(h.num_patterns >= 1 && h.num_patterns <= 9 && (h.required == 0 || h.required == 1));
    PG_CHECK_ARG(h.mask != nullptr && h.state != nullptr);
  }
  if (r->sampler == 1) {
    PG_CHECK_ARG(std::isfinite(r->temperature) && r->temperature >= 0.f && r->top_p > 0.f && r->top_p <= 1.f);
    PG_CHECK_ARG(r->top_k >= 0 && r->top_k <= r->V);
    PG_CHECK_ARG(r->sample_id != nullptr && r->end != nullptr && r->n_ended != nullptr && r->steps_run != nullptr);
  }
  if (r->nsteps == 0) return PROGEN_OK;
  cudaStream_t s = (cudaStream_t)stream;
  const bool bf = r->wdtype == PG_BF16;
  if (r->B == 1) return bf ? launch_run<1, bf16>(*r, s) : launch_run<1, float>(*r, s);
  if (r->B <= 8) return bf ? launch_run<8, bf16>(*r, s) : launch_run<8, float>(*r, s);
  // 9 .. 64 sequences: the 32-sequence tile, twice per phase above 32
  return bf ? launch_run<32, bf16>(*r, s) : launch_run<32, float>(*r, s);
}

}  // extern "C"
