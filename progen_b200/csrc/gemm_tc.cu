// wgmma GEMM for sm_90a: D[M,N] (+)= A[M,K] * B[N,K]^T, bf16 operands, fp32 accumulation in registers.
//
// Persistent and warp-specialized: min(tiles, SMs) CTAs, CTA b takes the 128 x 128 output tiles b, b + grid, b + 2 grid, ...
//   warpgroup 0    : TMA producer (one thread: cp.async.bulk.tensor.2d, 128B swizzle, mbarrier complete_tx); it walks
//                    the CTA's tiles with one ring position, so the next tile's k-blocks load during the epilogues
//   warpgroups 1, 2: ping-pong consumers: each owns whole tiles (alternate tiles of the CTA's list), two
//                    wgmma.mma_async m64n128k16 per k-step (both operands from shared memory), then the fused epilogue.
//                    A named-barrier handshake lets one warpgroup issue MMAs at a time, so one warpgroup's mainloop
//                    runs while the other is in its epilogue.
//
// Operands may be K-major or MN-major (wgrad reads the activations and the output gradient with the token dimension as
// K, i.e. MN-major): TMA writes both into the same 128B-swizzled layout and only the wgmma descriptors and transpose bits
// differ.  After the last k-block the accumulators go through a per-warpgroup shared-memory buffer, 64 rows at a time,
// so that every epilogue thread owns 8 consecutive columns of one row: the global loads / stores of the epilogue are
// 16-byte vectors, coalesced along the row.
#include <cuda.h>
#include <algorithm>
#include <mutex>
#include <unordered_map>
#include "gemm.h"
#include "tc_ptx.cuh"

namespace {

using namespace tc;

constexpr int BM = 128;
constexpr int BN = 128;
constexpr int BK = 64;                 // 64 bf16 = 128 bytes = one swizzle row
constexpr int WG_K = 16;               // K of one wgmma
constexpr int THREADS = 384;           // producer warpgroup + two consumer warpgroups
constexpr int A_BYTES = BM * BK * 2;   // 16 KiB
constexpr int B_BYTES = BN * BK * 2;   // 16 KiB
constexpr int STAGE_BYTES = A_BYTES + B_BYTES;
constexpr int STAGES = 4;                // a fifth stage fits only with epilogue passes of 64 x 64; measured slower on the step
constexpr int EPI_ROWS = 64;           // the epilogue stages and applies the tile in two passes of 64 rows
constexpr int EPI_ITEMS = EPI_ROWS * (BN / 8) / 128;   // row slices of 8 columns per consumer thread and pass
constexpr int CS_LD = BN + 4;          // fp32 row stride of the staged accumulator rows
constexpr int CS_BYTES = EPI_ROWS * CS_LD * 4;
constexpr int SMEM_TOTAL = 1024 /*align slack*/ + STAGES * STAGE_BYTES + 2 * CS_BYTES + 2 * STAGES * 8;
static_assert(SMEM_TOTAL <= 227 * 1024, "H100: 227 KiB of shared memory per block");
// named barriers (0 is __syncthreads): MMA turn of consumer c = 1 + c, epilogue buffer of consumer c = 3 + c
constexpr int BAR_TURN = 1, BAR_EPI = 3;
constexpr int PRODUCER_REGS = 40, CONSUMER_REGS = 232;     // setmaxnreg: 128 x 40 + 256 x 232 <= 64 K registers
static_assert(128 * PRODUCER_REGS + 256 * CONSUMER_REGS <= 65536, "register file");

__device__ __forceinline__ void named_bar_sync(int id, int n) { asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(n) : "memory"); }
__device__ __forceinline__ void named_bar_arrive(int id, int n) { asm volatile("bar.arrive %0, %1;" ::"r"(id), "r"(n) : "memory"); }
template <int R> __device__ __forceinline__ void setmaxnreg_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(R)); }
template <int R> __device__ __forceinline__ void setmaxnreg_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(R)); }

struct GemmDev {
  int M, N, K;
  int batch, batch_reduce;
  int a_batch_rows, b_batch_rows;
  long long d_batch_rows;
  int causal, split_k;
  EpiArgs epi;
  int K2;                              // tail operand pair: k-blocks of (A2, B2) after those of (A, B)
};

struct TileInfo {
  int z, m0, n0, kb_begin, kb_end;
  int kb_main;                         // TAIL: k-blocks kb_main .. kb_end - 1 are the tail's
};

template <bool TAIL>
__device__ __forceinline__ void decode_tile(const GemmDev& g, int t, TileInfo& ti) {
  const int m_tiles = (g.M + BM - 1) / BM;
  const int n_tiles = (g.N + BN - 1) / BN;
  const int per_z = g.split_k * m_tiles * n_tiles;
  ti.z = t / per_z;
  int r = t - ti.z * per_z;
  const int ks = r / (m_tiles * n_tiles);
  r -= ks * (m_tiles * n_tiles);
  ti.m0 = (r / n_tiles) * BM;
  ti.n0 = (r % n_tiles) * BN;
  const int kb_total = (g.K + BK - 1) / BK;
  int b = 0, e = kb_total;
  if (g.causal == 1) e = min(kb_total, (ti.m0 + BM + BK - 1) / BK);
  if (g.causal == 2) b = min(kb_total, ti.m0 / BK);
  if (g.split_k > 1) {
    const int per = (kb_total + g.split_k - 1) / g.split_k;
    b = min(kb_total, ks * per);
    e = min(kb_total, b + per);
  }
  ti.kb_begin = b;
  ti.kb_end = e;
  if constexpr (TAIL) {                // no split / causal / batch with a tail: (b, e) = (0, kb_total)
    ti.kb_main = e;
    ti.kb_end = e + (g.K2 + BK - 1) / BK;
  }
}

template <bool A_MN, bool B_MN, int KIND, typename TO, bool TAIL>
__global__ void __launch_bounds__(THREADS, 1)
gemm_tc_kernel(const __grid_constant__ CUtensorMap tma_a, const __grid_constant__ CUtensorMap tma_b,
               const __grid_constant__ CUtensorMap tma_a2, const __grid_constant__ CUtensorMap tma_b2, const GemmDev g,
               const int tiles) {
  extern __shared__ uint8_t smem_raw[];
  const uint32_t raw_u32 = smem_u32(smem_raw);
  const uint32_t smem_base = (raw_u32 + 1023u) & ~1023u;      // SWIZZLE_128B needs 1024 B alignment
  const uint32_t cs_base = smem_base + STAGES * STAGE_BYTES;
  const uint32_t bar_base = cs_base + 2 * CS_BYTES;
  auto full_bar = [&](int s) { return bar_base + 8u * s; };
  auto empty_bar = [&](int s) { return bar_base + 8u * (STAGES + s); };

  const int wg = threadIdx.x >> 7;
  if (threadIdx.x == 0) {
    prefetch_tensormap(&tma_a);
    prefetch_tensormap(&tma_b);
    if constexpr (TAIL) {
      prefetch_tensormap(&tma_a2);
      prefetch_tensormap(&tma_b2);
    }
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(full_bar(s), 1);
      mbar_init(empty_bar(s), 1);                 // released by the one consumer warpgroup that read the stage
    }
    fence_barrier_init();
  }
  __syncthreads();

  // The ring position runs on across tiles: the producer and both consumers see the same sequence of k-blocks (the
  // CTA's tiles in order), each consumer reading only its own tiles' k-blocks and stepping over the other's.
  int stage = 0;
  uint32_t phase = 0;
  auto advance = [&](int n) {
    stage += n;
    phase ^= (uint32_t)(stage / STAGES) & 1u;
    stage %= STAGES;
  };

  if (wg == 0) {
    // ===================================================================== TMA producer
    setmaxnreg_dec<PRODUCER_REGS>();
    if (threadIdx.x == 0) {
      for (int t = blockIdx.x; t < tiles; t += gridDim.x) {
        TileInfo ti;
        decode_tile<TAIL>(g, t, ti);
        const int a_row0 = ti.z * g.a_batch_rows;
        const int b_row0 = ti.z * g.b_batch_rows;
        for (int kb = ti.kb_begin; kb < ti.kb_end; ++kb) {
          mbar_wait(empty_bar(stage), phase ^ 1);
          const uint32_t sa = smem_base + stage * STAGE_BYTES;
          const uint32_t sb = sa + A_BYTES;
          mbar_expect_tx(full_bar(stage), STAGE_BYTES);
          if (TAIL && kb >= ti.kb_main) {
            // the tail pair (batch 1: row offset 0); TMA zero-fills the k-block beyond K2
            const int k0 = (kb - ti.kb_main) * BK;
            if constexpr (!A_MN) {
              tma_load_2d(sa, &tma_a2, full_bar(stage), k0, ti.m0);
            } else {
#pragma unroll
              for (int i = 0; i < BM / 64; ++i) tma_load_2d(sa + i * 8192, &tma_a2, full_bar(stage), ti.m0 + 64 * i, k0);
            }
            if constexpr (!B_MN) {
              tma_load_2d(sb, &tma_b2, full_bar(stage), k0, ti.n0);
            } else {
#pragma unroll
              for (int i = 0; i < BN / 64; ++i) tma_load_2d(sb + i * 8192, &tma_b2, full_bar(stage), ti.n0 + 64 * i, k0);
            }
            advance(1);
            continue;
          }
          const int k0 = kb * BK;
          if constexpr (!A_MN) {
            tma_load_2d(sa, &tma_a, full_bar(stage), k0, a_row0 + ti.m0);                   // box {64 k, 128 m}
          } else {
#pragma unroll
            for (int i = 0; i < BM / 64; ++i)                                                // boxes {64 m, 64 k}
              tma_load_2d(sa + i * 8192, &tma_a, full_bar(stage), ti.m0 + 64 * i, a_row0 + k0);
          }
          if constexpr (!B_MN) {
            tma_load_2d(sb, &tma_b, full_bar(stage), k0, b_row0 + ti.n0);                   // box {64 k, 128 n}
          } else {
#pragma unroll
            for (int i = 0; i < BN / 64; ++i)                                                // boxes {64 n, 64 k}
              tma_load_2d(sb + i * 8192, &tma_b, full_bar(stage), ti.n0 + 64 * i, b_row0 + k0);
          }
          advance(1);
        }
      }
    }
    return;
  }

  // ======================================================================= consumer c: tiles at even / odd positions
  setmaxnreg_inc<CONSUMER_REGS>();
  const int c = wg - 1;
  const int tid = threadIdx.x & 127;
  float* cs = reinterpret_cast<float*>(smem_raw + (cs_base - raw_u32)) + c * (CS_BYTES / 4);
  for (int p = 0, t = blockIdx.x; t < tiles; ++p, t += gridDim.x) {
    TileInfo ti;
    decode_tile<TAIL>(g, t, ti);
    if ((p & 1) != c) {
      advance(ti.kb_end - ti.kb_begin);
      continue;
    }
    // acc[h]: rows 64 h .. 64 h + 63 of the tile
    float acc[2][64];
#pragma unroll
    for (int i = 0; i < 64; ++i) acc[0][i] = acc[1][i] = 0.f;
    if (p > 0) named_bar_sync(BAR_TURN + c, 256);          // the other consumer has issued the MMAs of tile p - 1
    int prev = -1;
    for (int kb = ti.kb_begin; kb < ti.kb_end; ++kb) {
      mbar_wait(full_bar(stage), phase);
      const uint32_t sa = smem_base + stage * STAGE_BYTES;
      // both majors: rows 64 .. 127 of A start 8 KiB in (K-major: 64 rows x 128 B; MN-major: the second box)
      const uint64_t adesc0 = make_smem_desc<A_MN>(sa), adesc1 = make_smem_desc<A_MN>(sa + 8192);
      const uint64_t bdesc = make_smem_desc<B_MN>(sa + A_BYTES);
      constexpr uint32_t a_step = A_MN ? (2048 >> 4) : (32 >> 4), b_step = B_MN ? (2048 >> 4) : (32 >> 4);
      fence_regs(acc[0]);
      fence_regs(acc[1]);
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < BK / WG_K; ++k) {
        wgmma_m64n128k16_bf16<A_MN ? 1 : 0, B_MN ? 1 : 0>(acc[0], adesc0 + (uint64_t)(k * a_step), bdesc + (uint64_t)(k * b_step));
        wgmma_m64n128k16_bf16<A_MN ? 1 : 0, B_MN ? 1 : 0>(acc[1], adesc1 + (uint64_t)(k * a_step), bdesc + (uint64_t)(k * b_step));
      }
      wgmma_commit();
      fence_regs(acc[0]);
      fence_regs(acc[1]);
      wgmma_wait<1>();                          // the previous k-block's MMAs are done: its stage can be refilled
      if (prev >= 0 && tid == 0) mbar_arrive(empty_bar(prev));
      prev = stage;
      advance(1);
    }
    if (t + (int)gridDim.x < tiles) named_bar_arrive(BAR_TURN + (c ^ 1), 256);   // tile p + 1 may issue its MMAs

    // ---- epilogue, 64 rows per pass: stage the fp32 rows in this warpgroup's buffer, then 8 consecutive columns of
    // one row per thread, 16 threads per row.  Item i of pass h is tile row 64 h + 8 i + tid / 16, columns
    // 8 (tid % 16) .. + 7: a thread keeps its columns for the whole tile.  The global reads of a pass (epi_load) all go
    // out before its first item is finished, so a thread has EPI_ITEMS of them in flight instead of one.
    const int w = tid >> 5, lane = tid & 31;
    const int r0 = 16 * w + (lane >> 2), c0 = 2 * (lane & 3);
    const int cc = 8 * (tid & 15), col = ti.n0 + cc;
    const bool col_ok = col < g.N;
    const int m_first = ti.m0 + (tid >> 4);
    const long long row_first = (g.batch_reduce ? 0 : (long long)ti.z * g.d_batch_rows) + m_first;
    using CS = EpiColsum<KIND, 8>;
    EpiCol<8> cb;
    EpiPre<KIND, TO, 8> pre[EPI_ITEMS];
    epi_load_col<KIND, 8>(g.epi, col, col_ok, cb);
    // pass 0's load phase does not read the accumulators: it overlaps the last k-block's MMAs.  The residual kind
    // (64 prefetch registers and the bias) does not fit next to all 128 accumulators without spilling: it issues pass
    // 0's loads once acc[0] is staged.
    constexpr bool LOAD_BEFORE_WAIT = KIND != EPI_RESIDUAL;
    auto load_pass0 = [&] {
#pragma unroll
      for (int i = 0; i < EPI_ITEMS; ++i)
        epi_load<KIND, TO, 8>(g.epi, row_first + 8 * i, col, col_ok && m_first + 8 * i < g.M, pre[i]);
    };
    if constexpr (LOAD_BEFORE_WAIT) load_pass0();
    wgmma_wait<0>();
    fence_regs(acc[0]);
    fence_regs(acc[1]);
    if (prev >= 0 && tid == 0) mbar_arrive(empty_bar(prev));

    float csum[CS::REGS];
#pragma unroll
    for (int k = 0; k < CS::REGS; ++k) csum[k] = 0.f;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      named_bar_sync(BAR_EPI + c, 128);         // every thread has read the rows staged before
#pragma unroll
      for (int j = 0; j < BN / 8; ++j) {
        *reinterpret_cast<float2*>(cs + r0 * CS_LD + 8 * j + c0) = make_float2(acc[h][4 * j], acc[h][4 * j + 1]);
        *reinterpret_cast<float2*>(cs + (r0 + 8) * CS_LD + 8 * j + c0) = make_float2(acc[h][4 * j + 2], acc[h][4 * j + 3]);
      }
      if constexpr (!LOAD_BEFORE_WAIT) {
        if (h == 0) load_pass0();
      }
      named_bar_sync(BAR_EPI + c, 128);
#pragma unroll
      for (int i = 0; i < EPI_ITEMS; ++i) {
        const int r = 8 * i + (tid >> 4);
        const int m = m_first + EPI_ROWS * h + 8 * i;
        float v[8];
        const float4 x0 = *reinterpret_cast<const float4*>(cs + r * CS_LD + cc);
        const float4 x1 = *reinterpret_cast<const float4*>(cs + r * CS_LD + cc + 4);
        v[0] = x0.x; v[1] = x0.y; v[2] = x0.z; v[3] = x0.w; v[4] = x1.x; v[5] = x1.y; v[6] = x1.z; v[7] = x1.w;
        epi_finish<KIND, TO, 8>(g.epi, row_first + EPI_ROWS * h + 8 * i, col, v, cb, pre[i], col_ok && m < g.M, csum);
        // pass 1's load phase, one slot at a time as pass 0 frees it: in flight while pass 0 finishes and pass 1 stages
        if (h == 0)
          epi_load<KIND, TO, 8>(g.epi, row_first + EPI_ROWS + 8 * i, col, col_ok && m + EPI_ROWS < g.M, pre[i]);
      }
    }
    if constexpr (CS::W > 0) {
      if (g.epi.colsum) {                       // uniform
        // the tile's column sums: lanes l and l ^ 16 own the same columns; the four warps meet in the staging buffer,
        // then one red.global.add.v4 per 4 output columns
        constexpr int TW = 16 * CS::W;          // output columns of the tile
#pragma unroll
        for (int k = 0; k < CS::W; ++k) csum[k] += __shfl_xor_sync(0xffffffffu, csum[k], 16);
        named_bar_sync(BAR_EPI + c, 128);       // every thread has read the staged rows
        if (lane < 16) {
#pragma unroll
          for (int k = 0; k < CS::W; k += 4)
            *reinterpret_cast<float4*>(cs + w * TW + lane * CS::W + k) = make_float4(csum[k], csum[k + 1], csum[k + 2], csum[k + 3]);
        }
        named_bar_sync(BAR_EPI + c, 128);
        const int out0 = CS::OUT_SCALE * ti.n0, out_cols = CS::OUT_SCALE * g.N;
#pragma unroll
        for (int q = tid; q < TW / 4; q += 128) {
          float4 s = *reinterpret_cast<const float4*>(cs + 4 * q);
#pragma unroll
          for (int ww = 1; ww < 4; ++ww) {
            const float4 x = *reinterpret_cast<const float4*>(cs + ww * TW + 4 * q);
            s.x += x.x; s.y += x.y; s.z += x.z; s.w += x.w;
          }
          if (out0 + 4 * q < out_cols)
            asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(g.epi.colsum + out0 + 4 * q), "f"(s.x),
                         "f"(s.y), "f"(s.z), "f"(s.w) : "memory");
        }
      }
    }
  }
}

// ------------------------------------------------------------------------------------------ host side
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

EncodeTiledFn get_encode_fn() {
  static EncodeTiledFn fn = nullptr;
  static std::once_flag once;
  std::call_once(once, [] {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
        q == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<EncodeTiledFn>(p);
  });
  return fn;
}

struct MapKey {
  const void* ptr; uint64_t inner, outer, stride; uint32_t box_inner, box_outer, elem_bytes, swizzle;
  bool operator==(const MapKey& o) const {
    return ptr == o.ptr && inner == o.inner && outer == o.outer && stride == o.stride && box_inner == o.box_inner &&
           box_outer == o.box_outer && elem_bytes == o.elem_bytes && swizzle == o.swizzle;
  }
};
struct MapKeyHash {
  size_t operator()(const MapKey& k) const {
    size_t h = std::hash<const void*>()(k.ptr);
    auto mix = [&](uint64_t v) { h ^= std::hash<uint64_t>()(v) + 0x9e3779b97f4a7c15ULL + (h << 6) + (h >> 2); };
    mix(k.inner); mix(k.outer); mix(k.stride); mix(k.box_inner); mix(k.box_outer); mix(k.elem_bytes * 256 + k.swizzle);
    return h;
  }
};

// 2D tensor map: inner (contiguous) dimension first; elements of 2 (bf16) or 4 (fp32) bytes; swizzle span 32 / 64 /
// 128 bytes (= box_inner * elem_bytes for the epilogue boxes); OOB reads return zeros, OOB stores are clipped.
int get_tensor_map(const void* ptr, uint64_t inner, uint64_t outer, uint64_t row_stride_elems, uint32_t box_inner,
                   uint32_t box_outer, CUtensorMap* out, uint32_t elem_bytes = 2, uint32_t swizzle = 128) {
  static std::unordered_map<MapKey, CUtensorMap, MapKeyHash> cache;
  static std::mutex mu;
  MapKey key{ptr, inner, outer, row_stride_elems, box_inner, box_outer, elem_bytes, swizzle};
  std::lock_guard<std::mutex> lock(mu);
  auto it = cache.find(key);
  if (it != cache.end()) { *out = it->second; return PROGEN_OK; }
  EncodeTiledFn fn = get_encode_fn();
  if (!fn) { progen_set_error("cuTensorMapEncodeTiled driver entry point not found"); return PROGEN_ERR_DEVICE; }
  cuuint64_t dims[2] = {inner, outer};
  cuuint64_t strides[1] = {row_stride_elems * elem_bytes};
  const CUtensorMapSwizzle sw = swizzle == 128 ? CU_TENSOR_MAP_SWIZZLE_128B : swizzle == 64 ? CU_TENSOR_MAP_SWIZZLE_64B
                              : swizzle == 32 ? CU_TENSOR_MAP_SWIZZLE_32B : CU_TENSOR_MAP_SWIZZLE_NONE;
  cuuint32_t box[2] = {box_inner, box_outer};
  cuuint32_t estr[2] = {1, 1};
  CUtensorMap m;
  CUresult r = fn(&m, elem_bytes == 4 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT32 : CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2,
                  const_cast<void*>(ptr), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, sw, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    progen_set_error("cuTensorMapEncodeTiled failed (CUresult %d) ptr=%p inner=%llu outer=%llu stride=%llu box=%ux%u", (int)r,
                     ptr, (unsigned long long)inner, (unsigned long long)outer, (unsigned long long)row_stride_elems,
                     box_inner, box_outer);
    return PROGEN_ERR_CUDA;
  }
  if (cache.size() > 4096) cache.clear();
  cache.emplace(key, m);
  *out = m;
  return PROGEN_OK;
}


template <bool A_MN, bool B_MN, int KIND, typename TO, bool TAIL>
int launch_inst(const CUtensorMap& ta, const CUtensorMap& tb, const CUtensorMap& ta2, const CUtensorMap& tb2,
                const GemmDev& gd, int tiles, cudaStream_t stream) {
  auto kern = gemm_tc_kernel<A_MN, B_MN, KIND, TO, TAIL>;
  static bool attr_set = false;
  if (!attr_set) {
    PG_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_TOTAL));
    attr_set = true;
  }
  kern<<<std::min(tiles, pg_num_sms()), THREADS, SMEM_TOTAL, stream>>>(ta, tb, ta2, tb2, gd, tiles);
  PG_LAUNCH_CHECK();
  return PROGEN_OK;
}

}  // namespace

// shared with the wgmma attention kernels (attn_wgmma.cu)
int pg_tensor_map_2d_bf16(const void* ptr, uint64_t inner, uint64_t outer, uint64_t row_stride_elems, uint32_t box_inner,
                          uint32_t box_outer, CUtensorMap* out) {
  return get_tensor_map(ptr, inner, outer, row_stride_elems, box_inner, box_outer, out);
}

int gemm_tc_launch(const GemmArgs& a, cudaStream_t stream) {
  PG_CHECK_ARG(a.in_dtype == PG_BF16);
  PG_CHECK_ARG(a.M > 0 && a.N > 0 && a.K > 0 && a.batch >= 1 && a.split_k >= 1);
  PG_CHECK_ARG(a.N % 8 == 0);                        // 8-column epilogue items (an adapter's rank can be 8 .. 64)
  PG_CHECK_ARG(a.K % BK == 0);                       // TMA would zero-fill a K tail, but batched operands must not bleed
  PG_CHECK_ARG(a.lda % 8 == 0 && a.ldb % 8 == 0);    // 16-byte global strides for TMA
  PG_CHECK_ARG((reinterpret_cast<uintptr_t>(a.A) & 15) == 0 && (reinterpret_cast<uintptr_t>(a.B) & 15) == 0);
  PG_CHECK_ARG(!(a.split_k > 1 && a.causal));
  if (a.epi_kind == EPI_ROTARY) PG_CHECK_ARG(a.epi.seq_len % 32 == 0);
  PG_CHECK_ARG((reinterpret_cast<uintptr_t>(a.epi.colsum) & 15) == 0);    // red.global.add.v4
  PG_CHECK_ARG(!(a.split_k > 1 || a.batch_reduce) || (a.epi_kind == EPI_ACCUM && a.epi.atomic));
  PG_CHECK_TAIL(a);
  const bool tail = a.K2 > 0;
  if (tail) {
    PG_CHECK_ARG(a.K2 % 8 == 0 && a.lda2 % 8 == 0 && a.ldb2 % 8 == 0);
    PG_CHECK_ARG(a.a2_mn_major == a.a_mn_major && a.b2_mn_major == a.b_mn_major);
    PG_CHECK_ARG((reinterpret_cast<uintptr_t>(a.A2) & 15) == 0 && (reinterpret_cast<uintptr_t>(a.B2) & 15) == 0);
  }

  // stored 2D extents of each operand
  const uint64_t a_rows = (a.batch > 1 && a.a_batch_rows > 0) ? (uint64_t)a.a_batch_rows * a.batch
                                                              : (uint64_t)(a.a_mn_major ? a.K : a.M);
  const uint64_t b_rows = (a.batch > 1 && a.b_batch_rows > 0) ? (uint64_t)a.b_batch_rows * a.batch
                                                              : (uint64_t)(a.b_mn_major ? a.K : a.N);
  CUtensorMap ta, tb;
  int rc;
  if (!a.a_mn_major) rc = get_tensor_map(a.A, a.K, a_rows, a.lda, BK, BM, &ta);
  else               rc = get_tensor_map(a.A, a.M, a_rows, a.lda, 64, BK, &ta);
  if (rc) return rc;
  if (!a.b_mn_major) rc = get_tensor_map(a.B, a.K, b_rows, a.ldb, BK, BN, &tb);
  else               rc = get_tensor_map(a.B, a.N, b_rows, a.ldb, 64, BK, &tb);
  if (rc) return rc;
  CUtensorMap ta2 = ta, tb2 = tb;            // unused without a tail
  if (tail) {
    if (!a.a_mn_major) rc = get_tensor_map(a.A2, a.K2, a.M, a.lda2, BK, BM, &ta2);
    else               rc = get_tensor_map(a.A2, a.M, a.K2, a.lda2, 64, BK, &ta2);
    if (rc) return rc;
    if (!a.b_mn_major) rc = get_tensor_map(a.B2, a.K2, a.N, a.ldb2, BK, BN, &tb2);
    else               rc = get_tensor_map(a.B2, a.N, a.K2, a.ldb2, 64, BK, &tb2);
    if (rc) return rc;
  }

  GemmDev gd;
  gd.M = a.M; gd.N = a.N; gd.K = a.K;
  gd.batch = a.batch; gd.batch_reduce = a.batch_reduce;
  gd.a_batch_rows = (int)a.a_batch_rows; gd.b_batch_rows = (int)a.b_batch_rows; gd.d_batch_rows = a.d_batch_rows;
  gd.causal = a.causal; gd.split_k = a.split_k;
  gd.epi = a.epi;
  gd.K2 = a.K2;
  const long long tiles = (long long)a.batch * a.split_k * ((a.M + BM - 1) / BM) * ((a.N + BN - 1) / BN);
  PG_CHECK_ARG(tiles < (1ll << 31));

  const int am = a.a_mn_major ? 1 : 0, bm = a.b_mn_major ? 1 : 0;
  const bool obf = a.out_dtype == PG_BF16;
#define TC_CASE(AM, BMJ, KIND, TO)                                                                       \
  return tail ? launch_inst<AM, BMJ, KIND, TO, true>(ta, tb, ta2, tb2, gd, (int)tiles, stream)            \
              : launch_inst<AM, BMJ, KIND, TO, false>(ta, tb, ta2, tb2, gd, (int)tiles, stream)
  switch (a.epi_kind) {
    case EPI_STORE:
      if (!am && bm) { if (obf) TC_CASE(false, true, EPI_STORE, bf16); else TC_CASE(false, true, EPI_STORE, float); }
      if (!am && !bm) { if (obf) TC_CASE(false, false, EPI_STORE, bf16); else TC_CASE(false, false, EPI_STORE, float); }
      if (am && bm) { if (obf) TC_CASE(true, true, EPI_STORE, bf16); else TC_CASE(true, true, EPI_STORE, float); }
      break;
    case EPI_ROTARY:
      if (!am && bm && obf) TC_CASE(false, true, EPI_ROTARY, bf16);
      break;
    case EPI_RESIDUAL:
      if (!am && bm) TC_CASE(false, true, EPI_RESIDUAL, float);
      break;
    case EPI_GLU:
      if (!am && bm && obf) TC_CASE(false, true, EPI_GLU, bf16);
      break;
    case EPI_GELU:
      if (!am && bm && obf) TC_CASE(false, true, EPI_GELU, bf16);
      break;
    case EPI_GLU_BWD:
      if (!am && !bm && obf) TC_CASE(false, false, EPI_GLU_BWD, bf16);
      break;
    case EPI_GELU_BWD:
      if (!am && !bm && obf) TC_CASE(false, false, EPI_GELU_BWD, bf16);
      break;
    case EPI_ACCUM:
      // weight gradients take no tail (PG_CHECK_TAIL)
      if (am && bm) return launch_inst<true, true, EPI_ACCUM, float, false>(ta, tb, ta2, tb2, gd, (int)tiles, stream);
      if (!am && !bm) return launch_inst<false, false, EPI_ACCUM, float, false>(ta, tb, ta2, tb2, gd, (int)tiles, stream);
      break;
    default: break;
  }
#undef TC_CASE
  progen_set_error("gemm_tc: unsupported combination epi=%d a_mn=%d b_mn=%d out=%d", a.epi_kind, am, bm, a.out_dtype);
  return PROGEN_ERR_UNSUPPORTED;
}
