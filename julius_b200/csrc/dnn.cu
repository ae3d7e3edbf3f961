// dnn.cu -- K2: DNN-HMM forward for all frames of a batch on the Hopper tensor cores (wgmma).
//
// Stands in for dnn_calc_outprob (libsent/src/phmm/calc_dnn.c:774-868): per frame a stack of
//   dst = W.src + b   (calc_dnn_fma.c:18-95 / sub1 calc_dnn.c:509-523)
//   hidden: logistic through a 320001-entry table with clamps (calc_dnn.c:342-369)
//   output: linear, then log-softmax through addlog_array and "- log10 prior" (calc_dnn.c:862-865)
// The reference does this one frame at a time (a GEMV stack, 130 MB of weights per frame); here
// all frames of the batch go through one GEMM per layer:  C[frames x out] = A[frames x in] . W^T.
//
// Precision.  The parity tolerance is 1e-4 relative on log-likelihoods; a single bf16/tf32 pass
// (8/10-bit mantissa) is ~1e-3.  Every operand is therefore split in two bf16 terms
// (x = hi + lo, 16 mantissa bits) and each k-block issues three MMAs into the same fp32
// register accumulator:  hi.hi + hi.lo + lo.hi   (the dropped lo.lo term is 2^-16 relative).
//
// Kernel anatomy (sm_90a), dnn_gemm_wgmma: a persistent CTA per SM walks the 128 x 128 output tiles
// (column blocks fastest, so the CTAs that run side by side share the activation rows in L2).
// 384 threads = warpgroup 0 (one thread: the TMA producer) + two consumer warpgroups, each owning
// 64 rows of the tile.  Operand tiles 128 x 64 bf16 (K-major, 128-byte swizzle) arrive by
// cp.async.bulk.tensor (TMA) into a 3-stage shared-memory ring guarded by full/empty mbarriers
// (3 x 64 KB of the 227 KB a block may have).  The consumers issue wgmma.mma_async m64n128k16 straight
// from shared memory into 64 fp32 registers per thread, keep one wgmma group in flight while they
// wait for the next stage, and then run the epilogue from registers: bias, the reference's clamped
// table logistic, and the next layer's operands already split into bf16 hi/lo.  The producer runs
// ahead into the next tile meanwhile.  The last layer's epilogue writes fp32 logits; a row kernel then
// normalises them with a bit-exact replay of addlog_array (the reference's table-driven walk from the last
// output to the first) and subtracts the log10 prior.
#include "common.cuh"
#include <cuda.h>
#include <cuda_bf16.h>
#include <vector>
#include <cmath>

namespace jb200 {

static constexpr int BM = 128, BN = 128, BK = 64, STAGES = 3;
static constexpr int TILE_BYTES = BM * BK * 2;                 // 16 KB (A and B tiles are the same size)
static constexpr int STAGE_BYTES = 4 * TILE_BYTES;             // A_hi A_lo B_hi B_lo
static constexpr int CONSUMERS = 2;                            // warpgroups, 64 rows each
static constexpr int GEMM_THREADS = 128 * (1 + CONSUMERS);
static constexpr int GEMM_SMEM = STAGES * STAGE_BYTES + 1024 /*align*/ + 256 /*barriers*/;
static constexpr int LOGISTIC_N = 320001;

// ---- PTX wrappers ---------------------------------------------------------------------------------
__device__ __forceinline__ void tma_load_2d(void *dst, const CUtensorMap *map, uint64_t *bar, int c0, int c1) {
  asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
               :: "r"(smem_u32(dst)), "l"(map), "r"(smem_u32(bar)), "r"(c0), "r"(c1) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t *bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" :: "r"(smem_u32(bar)) : "memory");
}
// K-major, 128-byte swizzle wgmma matrix descriptor: start>>4 [0,14) | LBO=1 [16,30) (unused with this swizzle) |
// SBO=1024>>4 [32,46) (8 rows x 128 B) | layout SWIZZLE_128B=1 [62,64).  Tiles are 1024-byte aligned (base offset 0).
__device__ __forceinline__ uint64_t make_desc(const void *smem) {
  uint64_t d = (uint64_t)((smem_u32(smem) & 0x3ffff) >> 4);
  d |= (uint64_t)1 << 16;
  d |= (uint64_t)(1024 >> 4) << 32;
  d |= (uint64_t)1 << 62;
  return d;
}
__device__ __forceinline__ void wg_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wg_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" :: "n"(N) : "memory"); }
// D[64 x 128] (+)= A[64 x 16] . B[128 x 16]^T, bf16 in, fp32 accumulate; scale_d = 0 overwrites D
__device__ __forceinline__ void wgmma_bf16(float *d, uint64_t adesc, uint64_t bdesc, uint32_t scale_d) {
  asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
               "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 "
               "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63}, %64, %65, p, 1, 1, 0, 0;\n\t}"
               : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
               : "l"(adesc), "l"(bdesc), "r"(scale_d));
}

// logistic_func, calc_dnn.c:362-369
__device__ __forceinline__ float logistic_ref(float x, const float *__restrict__ tbl) {
  if (x <= -8.0f) return 0.000334f;
  if (x >= 8.0f) return 0.999666f;
  const float t = __fadd_rn(x, 8.0f);
  const int idx = (int)__dadd_rn((double)__fmul_rn(t, 20000.0f), 0.5);
  return __ldg(tbl + idx);
}

struct GemmArgs {
  int M, N, K;                 // rows (frames), outputs, inputs
  const float *bias;           // [N]
  const float *logistic;       // table
  __nv_bfloat16 *out_hi, *out_lo; int ld_out;   // hidden layers: next operands [M][ld_out]
  float *logits; int ld_logits;                 // last layer: fp32 [M][ld_logits]
  int last;
};

__global__ void __launch_bounds__(GEMM_THREADS, 1)
dnn_gemm_wgmma(const __grid_constant__ CUtensorMap map_a_hi, const __grid_constant__ CUtensorMap map_a_lo,
               const __grid_constant__ CUtensorMap map_b_hi, const __grid_constant__ CUtensorMap map_b_lo,
               const GemmArgs g) {
  extern __shared__ unsigned char dsm_raw[];
  unsigned char *dsm = reinterpret_cast<unsigned char *>((reinterpret_cast<uintptr_t>(dsm_raw) + 1023) & ~(uintptr_t)1023);
  uint64_t *full = reinterpret_cast<uint64_t *>(dsm + STAGES * STAGE_BYTES);
  uint64_t *empty = full + STAGES;

  const int wg = threadIdx.x >> 7, warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int nkb = (g.K + BK - 1) / BK;
  const int n_nblk = (g.N + BN - 1) / BN, n_mblk = (g.M + BM - 1) / BM;
  const int n_tiles = n_nblk * n_mblk;

  if (threadIdx.x == 0) {
    for (int s = 0; s < STAGES; s++) { mbar_init(&full[s], 1); mbar_init(&empty[s], CONSUMERS * 4); }
    mbar_fence_init();
  }
  __syncthreads();

  if (wg == 0) {
    if (threadIdx.x == 0) {
      // ===== TMA producer =====
      int it = 0;
      for (int tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
        const int m0 = (tile / n_nblk) * BM, n0 = (tile % n_nblk) * BN;
        for (int kb = 0; kb < nkb; kb++, it++) {
          const int s = it % STAGES;
          const uint32_t ph = (it / STAGES) & 1;
          mbar_wait(&empty[s], ph ^ 1);
          unsigned char *st = dsm + s * STAGE_BYTES;
          mbar_expect_tx(&full[s], STAGE_BYTES);
          tma_load_2d(st, &map_a_hi, &full[s], kb * BK, m0);
          tma_load_2d(st + TILE_BYTES, &map_a_lo, &full[s], kb * BK, m0);
          tma_load_2d(st + 2 * TILE_BYTES, &map_b_hi, &full[s], kb * BK, n0);
          tma_load_2d(st + 3 * TILE_BYTES, &map_b_lo, &full[s], kb * BK, n0);
        }
      }
    }
    return;
  }

  // ===== consumer warpgroups: rows [64*c, 64*c+64) of every tile =====
  const int c = wg - 1;
  const int wl = warp & 3;                                     // warp inside the warpgroup
  float d[64];
  int it = 0;
  for (int tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
    const int m0 = (tile / n_nblk) * BM, n0 = (tile % n_nblk) * BN;
    for (int kb = 0; kb < nkb; kb++, it++) {
      const int s = it % STAGES;
      mbar_wait(&full[s], (it / STAGES) & 1);
      unsigned char *st = dsm + s * STAGE_BYTES;
      const uint64_t a_hi = make_desc(st + c * (64 * 128)), a_lo = make_desc(st + TILE_BYTES + c * (64 * 128));
      const uint64_t b_hi = make_desc(st + 2 * TILE_BYTES), b_lo = make_desc(st + 3 * TILE_BYTES);
      wg_fence();
#pragma unroll
      for (int k = 0; k < BK / 16; k++) {
        const uint64_t adv = (uint64_t)(k * 32 >> 4);        // 16 bf16 = 32 bytes along K inside the swizzle atom
        wgmma_bf16(d, a_hi + adv, b_hi + adv, (kb | k) ? 1u : 0u);
        wgmma_bf16(d, a_hi + adv, b_lo + adv, 1u);
        wgmma_bf16(d, a_lo + adv, b_hi + adv, 1u);
      }
      wg_commit();
      // the previous k-block's group has retired once at most this one is pending: hand its stage back
      wg_wait<1>();
      if (kb > 0) {
        __syncwarp();
        if (lane == 0) mbar_arrive(&empty[(it - 1) % STAGES]);
      }
    }
    wg_wait<0>();
    __syncwarp();
    if (lane == 0) mbar_arrive(&empty[(it - 1) % STAGES]);

    // ===== epilogue from registers: element (row, col) of d[4j + 2h + e] is
    //       row = 16*wl + lane/4 + 8h, col = 8j + 2*(lane%4) + e =====
#pragma unroll
    for (int h = 0; h < 2; h++) {
      const int row = m0 + c * 64 + wl * 16 + (lane >> 2) + 8 * h;
      if (row >= g.M) continue;
#pragma unroll
      for (int j = 0; j < BN / 8; j++) {
        const int col = n0 + 8 * j + 2 * (lane & 3);
        const float x0 = d[4 * j + 2 * h], x1 = d[4 * j + 2 * h + 1];
        if (g.last) {
          float *dst = g.logits + (size_t)row * g.ld_logits + col;
          if (col < g.N) dst[0] = x0 + __ldg(g.bias + col);
          if (col + 1 < g.N) dst[1] = x1 + __ldg(g.bias + col + 1);
        } else if (col < g.ld_out) {
          // ld_out is a multiple of 8 and col even: col + 1 < ld_out too.  Columns beyond N (up to ld_out) are
          // written as zeros so the next layer's K tail is clean
          const float v0 = (col < g.N) ? logistic_ref(x0 + __ldg(g.bias + col), g.logistic) : 0.0f;
          const float v1 = (col + 1 < g.N) ? logistic_ref(x1 + __ldg(g.bias + col + 1), g.logistic) : 0.0f;
          const __nv_bfloat16 h0 = __float2bfloat16_rn(v0), h1 = __float2bfloat16_rn(v1);
          __nv_bfloat162 hi, lo;
          hi.x = h0; hi.y = h1;
          lo.x = __float2bfloat16_rn(v0 - __bfloat162float(h0));
          lo.y = __float2bfloat16_rn(v1 - __bfloat162float(h1));
          *reinterpret_cast<__nv_bfloat162 *>(g.out_hi + (size_t)row * g.ld_out + col) = hi;
          *reinterpret_cast<__nv_bfloat162 *>(g.out_lo + (size_t)row * g.ld_out + col) = lo;
        }
      }
    }
  }
}

// Layer 0's operand: network input rows [M][K] as bf16 hi/lo [M][ld] (zero padded).  Input row r, column c is column
// c % fl of frame c / fl of row r's window (SpliceSeg), so the operand is bit for bit that of the rows spliced on the
// host.  Without a segment table the window of row r is src frames r .. r + K / fl - 1, which lie back to back: column c
// is src[r * fl + c] (with context 1, fl == K, the plain row-major copy).
__global__ void split_bf16_kernel(const float *__restrict__ src, int fl, const SpliceMap sm, int M, int K, __nv_bfloat16 *hi,
                                  __nv_bfloat16 *lo, int ld) {
  const size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (size_t)M * ld) return;
  const int r = (int)(idx / ld), c = (int)(idx % ld);
  float v = 0.0f;
  if (c < K) {
    if (sm.nseg == 0) {
      v = src[(size_t)r * fl + c];
    } else {
      int a = 0, b = sm.nseg - 1;                              // the last segment whose rows start at or before r
      while (a < b) {
        const int m = (a + b + 1) >> 1;
        if (__ldg(&sm.seg[m].row0) <= r) a = m; else b = m - 1;
      }
      const SpliceSeg s = sm.seg[a];
      v = __ldg(splice_frame(s, r - s.row0 + c / fl, src, sm.carry, fl) + c % fl);
    }
  }
  const __nv_bfloat16 h = __float2bfloat16_rn(v);
  hi[idx] = h;
  lo[idx] = __float2bfloat16_rn(v - __bfloat162float(h));
}

// log-softmax + prior (calc_dnn.c:862-865).  The normaliser is addlog_array (addlog.c:102-123) replayed bit for bit:
// the outputs are walked from N-1 down to 0 into a running fp32 sum y (start LOG_ZERO), a term more than LOG_ADDMIN
// below y as it stands at that point of the walk is dropped, the others are added through the 500 000-entry table.
// That walk is a chain of dependent table loads, so each lane runs the chain of its own frame (a warp takes 32 frames);
// the warp stages 32 outputs of its 32 frames at a time through shared memory, read coalesced and transposed.  Then
// the warp writes each of its frames' score rows together.
static constexpr int SOFTMAX_WARPS = 4;
__global__ void __launch_bounds__(32 * SOFTMAX_WARPS)
dnn_softmax_kernel(const float *__restrict__ logits, int ld_logits, int N, int T, const float *__restrict__ prior,
                   const float *__restrict__ addlog_tbl, float *__restrict__ rows, int row_stride) {
  __shared__ float s_tile[SOFTMAX_WARPS][32][33];
  const int lane = threadIdx.x & 31;
  const int f0 = (blockIdx.x * SOFTMAX_WARPS + (threadIdx.x >> 5)) * 32;   // first frame of this warp
  if (f0 >= T) return;
  const int nf = min(32, T - f0);
  float (*tile)[33] = s_tile[threadIdx.x >> 5];
  float y = JB200_LOG_ZERO;
  for (int hi = N - 1; hi >= 0; hi -= 32) {
    // tile[r][c] = output hi - c of frame f0 + r: c is the position in the walk
    const int i = hi - lane;
    for (int r = 0; r < nf; r++) tile[r][lane] = (i >= 0) ? __ldg(logits + (size_t)(f0 + r) * ld_logits + i) : 0.0f;
    __syncwarp();
    const int cnt = min(32, hi + 1);
    if (lane < nf)
      for (int c = 0; c < cnt; c++) y = addlog_step_exact(y, tile[lane][c], addlog_tbl);
    __syncwarp();
  }
  for (int r = 0; r < nf; r++) {
    const float lp = __shfl_sync(0xffffffffu, y, r);
    const float *x = logits + (size_t)(f0 + r) * ld_logits;
    float *out = rows + (size_t)(f0 + r) * row_stride;
    for (int i = lane; i < N; i += 32)
      out[i] = (float)__dsub_rn(__dmul_rn(JB200_INV_LOG_TEN, (double)__fsub_rn(__ldg(x + i), lp)), (double)__ldg(prior + i));
  }
}

}  // namespace jb200

// =============================================================================================
using namespace jb200;

typedef CUresult (*PFN_encodeTiled)(CUtensorMap *, CUtensorMapDataType, cuuint32_t, void *, const cuuint64_t *, const cuuint64_t *,
                                    const cuuint32_t *, const cuuint32_t *, CUtensorMapInterleave, CUtensorMapSwizzle,
                                    CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

struct DnnLayerDev {
  int in = 0, out = 0, ld_in = 0;          // ld_in: K padded to a multiple of 8 (16-byte row pitch)
  __nv_bfloat16 *w_hi = nullptr, *w_lo = nullptr;   // [out][ld_in]
  float *bias = nullptr;
  CUtensorMap map_w_hi, map_w_lo;
};

struct jb200_dnn {
  int device = 0, n_layers = 0, in_dim = 0, out_dim = 0, row_stride = 0;
  // input frames are frame_len = in_dim / context wide, spliced context at a time (jb200_dnn_set_context); fixed once
  // the handle has scored frames or been attached to a decoder
  int context = 1, frame_len = 0; bool layout_fixed = false;
  std::vector<DnnLayerDev> L;
  float *d_prior = nullptr, *d_logistic = nullptr, *d_addlog = nullptr;
  PFN_encodeTiled encode = nullptr;
  cudaStream_t stream = nullptr;
  // batch buffers
  int cap_frames = 0, max_width = 0, ld_logits = 0, n_sm = 0;
  float *d_in = nullptr, *d_logits = nullptr, *d_rows = nullptr;
  __nv_bfloat16 *act_hi[2] = {nullptr, nullptr}, *act_lo[2] = {nullptr, nullptr};
  // the end of the last forward: the next one waits for it on its own stream, since every forward uses the buffers above
  // and decoders (or a decoder group) sharing the handle call it on different streams
  cudaEvent_t forward_done = nullptr;
};

static int make_map(jb200_dnn *h, CUtensorMap *map, void *base, int rows, int cols_ld, int cols_valid) {
  // 2-D bf16 tensor [rows][cols_ld], box = {64 columns (128 B), 128 rows}, 128-byte swizzle, OOB -> zeros
  cuuint64_t gdim[2] = {(cuuint64_t)cols_valid, (cuuint64_t)rows};
  cuuint64_t gstr[1] = {(cuuint64_t)cols_ld * 2};
  cuuint32_t box[2] = {(cuuint32_t)BK, (cuuint32_t)BM};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = h->encode(map, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, base, gdim, gstr, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                         CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) { set_error("cuTensorMapEncodeTiled failed (%d) rows=%d ld=%d", (int)r, rows, cols_ld); return JB200_ERR_CUDA; }
  return JB200_OK;
}

extern "C" void jb200_dnn_destroy(jb200_dnn *h) {
  if (!h) return;
  cudaSetDevice(h->device);
  for (auto &l : h->L) { cudaFree(l.w_hi); cudaFree(l.w_lo); cudaFree(l.bias); }
  cudaFree(h->d_prior); cudaFree(h->d_logistic); cudaFree(h->d_addlog); cudaFree(h->d_in); cudaFree(h->d_logits); cudaFree(h->d_rows);
  for (int i = 0; i < 2; i++) { cudaFree(h->act_hi[i]); cudaFree(h->act_lo[i]); }
  if (h->forward_done) cudaEventDestroy(h->forward_done);
  if (h->stream) cudaStreamDestroy(h->stream);
  delete h;
}

// the device half of jb200_dnn_create
static int dnn_build(jb200_dnn *h, const jb200_dnn_desc *d) {
  {
    void *fn = nullptr; cudaDriverEntryPointQueryResult qres;
    cudaError_t e = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &qres);
    if (e != cudaSuccess || qres != cudaDriverEntryPointSuccess || !fn) { set_error("cuTensorMapEncodeTiled not available"); return JB200_ERR_CUDA; }
    h->encode = (PFN_encodeTiled)fn;
  }
  JB_CUDA(cudaStreamCreateWithFlags(&h->stream, cudaStreamNonBlocking));
  h->L.resize(d->n_layers);
  h->max_width = (d->in_dim + 7) & ~7;
  for (int l = 0; l < d->n_layers; l++) {
    DnnLayerDev &L = h->L[l];
    L.in = d->layer_in[l]; L.out = d->layer_out[l]; L.ld_in = (L.in + 7) & ~7;
    if (l + 1 < d->n_layers) h->max_width = std::max(h->max_width, (L.out + 7) & ~7);
    std::vector<__nv_bfloat16> hi((size_t)L.out * L.ld_in), lo((size_t)L.out * L.ld_in);
    for (int r = 0; r < L.out; r++)
      for (int c = 0; c < L.ld_in; c++) {
        const float v = (c < L.in) ? d->w[l][(size_t)r * L.in + c] : 0.0f;
        const __nv_bfloat16 b = __float2bfloat16_rn(v);
        hi[(size_t)r * L.ld_in + c] = b;
        lo[(size_t)r * L.ld_in + c] = __float2bfloat16_rn(v - __bfloat162float(b));
      }
    JB_CUDA(cudaMalloc(&L.w_hi, hi.size() * 2)); JB_CUDA(cudaMalloc(&L.w_lo, lo.size() * 2));
    JB_CUDA(cudaMemcpy(L.w_hi, hi.data(), hi.size() * 2, cudaMemcpyHostToDevice));
    JB_CUDA(cudaMemcpy(L.w_lo, lo.data(), lo.size() * 2, cudaMemcpyHostToDevice));
    JB_CUDA(cudaMalloc(&L.bias, sizeof(float) * L.out));
    JB_CUDA(cudaMemcpy(L.bias, d->b[l], sizeof(float) * L.out, cudaMemcpyHostToDevice));
    JB_RC(make_map(h, &L.map_w_hi, L.w_hi, L.out, L.ld_in, L.ld_in));
    JB_RC(make_map(h, &L.map_w_lo, L.w_lo, L.out, L.ld_in, L.ld_in));
  }
  JB_CUDA(cudaMalloc(&h->d_prior, sizeof(float) * d->out_dim));
  JB_CUDA(cudaMemcpy(h->d_prior, d->state_prior, sizeof(float) * d->out_dim, cudaMemcpyHostToDevice));
  {
    // logistic_table_build, calc_dnn.c:350-360
    std::vector<float> tbl(LOGISTIC_N);
    for (int i = 0; i < LOGISTIC_N; i++) { double x = (double)i / 20000.0 - 8.0; tbl[i] = (float)(1.0 / (1.0 + exp(-x))); }
    JB_CUDA(cudaMalloc(&h->d_logistic, sizeof(float) * LOGISTIC_N));
    JB_CUDA(cudaMemcpy(h->d_logistic, tbl.data(), sizeof(float) * LOGISTIC_N, cudaMemcpyHostToDevice));
    build_addlog_table(tbl);
    JB_CUDA(cudaMalloc(&h->d_addlog, sizeof(float) * tbl.size()));
    JB_CUDA(cudaMemcpy(h->d_addlog, tbl.data(), sizeof(float) * tbl.size(), cudaMemcpyHostToDevice));
  }
  h->ld_logits = (d->out_dim + 3) & ~3;
  JB_CUDA(cudaFuncSetAttribute(dnn_gemm_wgmma, cudaFuncAttributeMaxDynamicSharedMemorySize, GEMM_SMEM));
  return JB200_OK;
}

extern "C" int jb200_dnn_create(const jb200_dnn_desc *d, int device, jb200_dnn **out) {
  if (!d || !out || d->n_layers < 1 || d->n_layers > JB200_DNN_MAX_LAYERS) { set_error("jb200_dnn_create: bad argument"); return JB200_ERR_ARG; }
  // the kernels trust these: the input copy is in_dim wide, each layer reads what the one before wrote, the last layer
  // writes layer_out[n-1] columns into rows padded from out_dim, and the prior and the score rows are out_dim wide
  for (int l = 0; l < d->n_layers; l++) {
    if (d->layer_in[l] < 1 || d->layer_out[l] < 1) { set_error("jb200_dnn_create: layer %d is %d -> %d", l, d->layer_in[l], d->layer_out[l]); return JB200_ERR_ARG; }
    if (l > 0 && d->layer_in[l] != d->layer_out[l - 1]) { set_error("jb200_dnn_create: layer %d input %d != previous output %d", l, d->layer_in[l], d->layer_out[l - 1]); return JB200_ERR_ARG; }
  }
  if (d->in_dim != d->layer_in[0] || d->out_dim != d->layer_out[d->n_layers - 1]) {
    set_error("jb200_dnn_create: net is %d -> %d but its layers take %d and give %d", d->in_dim, d->out_dim, d->layer_in[0], d->layer_out[d->n_layers - 1]);
    return JB200_ERR_ARG;
  }
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev <= 0) { set_error("no CUDA device (libjb200 has no CPU fallback)"); return JB200_ERR_NODEVICE; }
  if (device < 0 || device >= ndev) { set_error("device %d out of range", device); return JB200_ERR_ARG; }
  JB_CUDA(cudaSetDevice(device));
  cudaDeviceProp prop;
  JB_CUDA(cudaGetDeviceProperties(&prop, device));
  if (prop.major != 9) { set_error("device is sm_%d%d; the wgmma GEMM needs sm_90a", prop.major, prop.minor); return JB200_ERR_NODEVICE; }
  jb200_dnn *h = new jb200_dnn();
  h->device = device; h->n_layers = d->n_layers; h->in_dim = d->in_dim; h->out_dim = d->out_dim; h->frame_len = d->in_dim;
  h->row_stride = (d->out_dim + 3) & ~3;
  h->n_sm = prop.multiProcessorCount;
  const int rc = dnn_build(h, d);
  if (rc) { jb200_dnn_destroy(h); return rc; }
  *out = h;
  return JB200_OK;
}

extern "C" int jb200_dnn_out_dim(const jb200_dnn *h) { return h ? h->out_dim : 0; }
extern "C" int jb200_dnn_in_dim(const jb200_dnn *h) { return h ? h->in_dim : 0; }

extern "C" int jb200_dnn_set_context(jb200_dnn *h, int context_len) {
  if (!h || context_len < 1) { set_error("jb200_dnn_set_context: bad argument"); return JB200_ERR_ARG; }
  if (h->in_dim % context_len) { set_error("jb200_dnn_set_context: input width %d is not a multiple of %d frames", h->in_dim, context_len); return JB200_ERR_ARG; }
  if (h->layout_fixed) { set_error("jb200_dnn_set_context: the handle has scored frames or been attached to a decoder"); return JB200_ERR_ARG; }
  h->context = context_len; h->frame_len = h->in_dim / context_len;
  return JB200_OK;
}

static int dnn_reserve(jb200_dnn *h, int T) {
  if (T <= h->cap_frames) return JB200_OK;
  cudaFree(h->d_in); cudaFree(h->d_logits); cudaFree(h->d_rows);
  for (int i = 0; i < 2; i++) { cudaFree(h->act_hi[i]); cudaFree(h->act_lo[i]); h->act_hi[i] = h->act_lo[i] = nullptr; }
  h->d_in = h->d_logits = h->d_rows = nullptr; h->cap_frames = 0;
  JB_CUDA(cudaMalloc(&h->d_in, sizeof(float) * (size_t)T * h->in_dim));
  JB_CUDA(cudaMalloc(&h->d_logits, sizeof(float) * (size_t)T * h->ld_logits));
  JB_CUDA(cudaMalloc(&h->d_rows, sizeof(float) * (size_t)T * h->row_stride));
  for (int i = 0; i < 2; i++) {
    JB_CUDA(cudaMalloc(&h->act_hi[i], 2 * (size_t)T * h->max_width));
    JB_CUDA(cudaMalloc(&h->act_lo[i], 2 * (size_t)T * h->max_width));
  }
  h->cap_frames = T;
  return JB200_OK;
}

namespace jb200 {
// the decoder's view of the handle: from now on its input layout stays as it is; returns the context length
int dnn_fix_context(jb200_dnn *h) {
  h->layout_fixed = true;
  return h->context;
}

// T network input rows, each the window of context frames (frame_len floats each) that sm gives for it, from d_in
// (fp32, device) -> d_rows [T][row_stride] log10 pseudo-likelihoods
int dnn_forward_device(jb200_dnn *h, const float *d_in, int T, float *d_rows, int row_stride, cudaStream_t st, const SpliceMap &sm) {
  if (T <= 0) return JB200_OK;
  JB_CUDA(cudaSetDevice(h->device));
  int rc = dnn_reserve(h, T); if (rc) return rc;
  if (!h->forward_done) JB_CUDA(cudaEventCreateWithFlags(&h->forward_done, cudaEventDisableTiming));
  JB_CUDA(cudaStreamWaitEvent(st, h->forward_done, 0));
  int cur = 0;
  {
    const int ld = h->L[0].ld_in;
    const size_t tot = (size_t)T * ld;
    split_bf16_kernel<<<(unsigned)((tot + 255) / 256), 256, 0, st>>>(d_in, h->frame_len, sm, T, h->in_dim, h->act_hi[0], h->act_lo[0], ld);
    JB_LAUNCH_CHECK();
  }
  for (int l = 0; l < h->n_layers; l++) {
    DnnLayerDev &L = h->L[l];
    CUtensorMap ma_hi, ma_lo;
    rc = make_map(h, &ma_hi, h->act_hi[cur], T, L.ld_in, L.ld_in); if (rc) return rc;
    rc = make_map(h, &ma_lo, h->act_lo[cur], T, L.ld_in, L.ld_in); if (rc) return rc;
    GemmArgs g;
    g.M = T; g.N = L.out; g.K = L.ld_in; g.bias = L.bias; g.logistic = h->d_logistic;
    g.last = (l + 1 == h->n_layers) ? 1 : 0;
    g.out_hi = h->act_hi[cur ^ 1]; g.out_lo = h->act_lo[cur ^ 1];
    g.ld_out = g.last ? 0 : h->L[l + 1].ld_in;
    g.logits = h->d_logits; g.ld_logits = h->ld_logits;
    const int tiles = ((L.out + BN - 1) / BN) * ((T + BM - 1) / BM);
    dnn_gemm_wgmma<<<std::min(tiles, h->n_sm), GEMM_THREADS, GEMM_SMEM, st>>>(ma_hi, ma_lo, L.map_w_hi, L.map_w_lo, g);
    JB_LAUNCH_CHECK();
    cur ^= 1;
  }
  dnn_softmax_kernel<<<(T + 32 * SOFTMAX_WARPS - 1) / (32 * SOFTMAX_WARPS), 32 * SOFTMAX_WARPS, 0, st>>>(h->d_logits, h->ld_logits, h->out_dim, T,
                                                                                        h->d_prior, h->d_addlog, d_rows, row_stride);
  JB_LAUNCH_CHECK();
  JB_CUDA(cudaEventRecord(h->forward_done, st));
  return JB200_OK;
}
}  // namespace jb200

// n_frames input frames give n_frames - context + 1 rows (none when the input is shorter than the window); the input
// copy, (T + context - 1) * frame_len floats, fits in the T * in_dim that dnn_reserve gives d_in
extern "C" int jb200_dnn_score_host(jb200_dnn *h, const float *in, int n_frames, float *scores) {
  if (!h || !in || !scores) { set_error("jb200_dnn_score_host: null argument"); return JB200_ERR_ARG; }
  h->layout_fixed = true;
  const int T = n_frames - h->context + 1;
  if (T <= 0) return JB200_OK;
  JB_CUDA(cudaSetDevice(h->device));
  int rc = dnn_reserve(h, T); if (rc) return rc;
  JB_CUDA(cudaMemcpyAsync(h->d_in, in, sizeof(float) * (size_t)n_frames * h->frame_len, cudaMemcpyHostToDevice, h->stream));
  rc = dnn_forward_device(h, h->d_in, T, h->d_rows, h->row_stride, h->stream, SpliceMap()); if (rc) return rc;
  JB_CUDA(cudaMemcpy2DAsync(scores, sizeof(float) * h->out_dim, h->d_rows, sizeof(float) * h->row_stride, sizeof(float) * h->out_dim, T,
                            cudaMemcpyDeviceToHost, h->stream));
  JB_CUDA(cudaStreamSynchronize(h->stream));
  return JB200_OK;
}
