// Host side of the wgmma GEMM family: TMA tensor-map construction, tile mapping and launch.
#include <stdarg.h>

#include <algorithm>
#include <mutex>

#include "../../include/unispeech_b200.h"
#include "common.h"
#include "gemm.cuh"

namespace b200 {

// ------------------------------------------------------------------ error plumbing
long long g_launch_count = 0;
static thread_local char g_err[512] = "";
char* last_error_buf() { return g_err; }
void set_last_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}
int sm_count() {
  static int n = 0;
  if (n == 0) {
    int dev = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev);
    if (n <= 0) n = 132;
  }
  return n;
}

// ------------------------------------------------------------------ tensor maps
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
static EncodeTiledFn get_encode_fn() {
  static EncodeTiledFn fn = nullptr;
  static std::once_flag once;
  std::call_once(once, [] {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres) == cudaSuccess &&
        qres == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<EncodeTiledFn>(p);
  });
  return fn;
}

struct ViewSpec {
  const void* ptr;
  long long dims[4];     // elements; dims[0] contiguous
  long long strides[3];  // elements, for dims 1..3
  int box[4];
  CUtensorMapDataType dtype = CU_TENSOR_MAP_DATA_TYPE_BFLOAT16;
  CUtensorMapSwizzle swizzle = CU_TENSOR_MAP_SWIZZLE_128B;
};

// bf16, fp32 or bytes (fp8), zero OOB fill; bf16 and byte maps (MMA operands) promote 256-byte L2 lines, fp32 maps (reduction destinations) none.
// Returns 0 on success.
static int make_tmap(CUtensorMap* out, const ViewSpec& v) {
  EncodeTiledFn fn = get_encode_fn();
  if (!fn) {
    set_last_error("cuTensorMapEncodeTiled entry point not available (no CUDA driver?)");
    return -3;
  }
  const bool f32 = v.dtype == CU_TENSOR_MAP_DATA_TYPE_FLOAT32;
  const long long esize = f32 ? 4 : v.dtype == CU_TENSOR_MAP_DATA_TYPE_UINT8 ? 1 : 2;
  cuuint64_t dims[4];
  cuuint64_t strides[3];
  cuuint32_t box[4];
  cuuint32_t estr[4] = {1, 1, 1, 1};
  for (int i = 0; i < 4; ++i) {
    dims[i] = static_cast<cuuint64_t>(v.dims[i] > 0 ? v.dims[i] : 1);
    box[i] = static_cast<cuuint32_t>(v.box[i]);
  }
  for (int i = 0; i < 3; ++i) {
    long long s = v.strides[i];
    if (s <= 0) s = (i == 0 ? v.dims[0] : static_cast<long long>(strides[i - 1] / esize) * v.dims[i]);
    if (s * esize % 16 != 0) {
      set_last_error("tensor map stride %lld (dim %d) is not a multiple of 16 bytes", s, i + 1);
      return -1;
    }
    strides[i] = static_cast<cuuint64_t>(s * esize);
  }
  if ((reinterpret_cast<uintptr_t>(v.ptr) & 15) != 0) {
    set_last_error("tensor map base pointer %p is not 16-byte aligned", v.ptr);
    return -1;
  }
  CUresult r = fn(out, v.dtype, 4, const_cast<void*>(v.ptr), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, v.swizzle,
                  f32 ? CU_TENSOR_MAP_L2_PROMOTION_NONE : CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_last_error("cuTensorMapEncodeTiled failed (%d): dims {%lld,%lld,%lld,%lld} strides {%lld,%lld,%lld} box {%d,%d,%d,%d}",
                   static_cast<int>(r), v.dims[0], v.dims[1], v.dims[2], v.dims[3], v.strides[0], v.strides[1],
                   v.strides[2], v.box[0], v.box[1], v.box[2], v.box[3]);
    return -3;
  }
  return 0;
}

// [B, T, cols] bf16 or fp32 row-major seen as [B, T, cols / hd heads, hd] (innermost dimension = one attention head): box =
// box_cols columns of one head x box_rows rows, addressed by (column in the head, head slot, row, batch).  A load box that
// reaches past the head's last column gets zeros there, and a reduction box is clipped there (and at T), so no column of a
// neighbouring head is read or written (the attention kernels' operands and dQ accumulator).
int make_head_tmap(CUtensorMap* out, const void* ptr, CUtensorMapDataType dtype, int T, int B, int cols, int hd, int box_cols,
                   int box_rows, CUtensorMapSwizzle swizzle) {
  ViewSpec v{ptr, {hd, cols / hd, T, B}, {hd, cols, static_cast<long long>(T) * cols}, {box_cols, 1, box_rows, 1}, dtype, swizzle};
  return make_tmap(out, v);
}

// [batches, rows, cols] bf16 with arbitrary row / batch strides (elements): box = 64 columns x box_rows rows (k-means operands)
int make_rows_tmap(CUtensorMap* out, const void* ptr, long long cols, long long rows, long long batches, long long row_stride,
                   long long batch_stride, int box_rows) {
  ViewSpec v{ptr, {cols, rows, batches, 1}, {row_stride, batches > 1 ? batch_stride : 0, 0}, {64, box_rows, 1, 1}};
  return make_tmap(out, v);
}

// [batches, rows, K] e4m3 bytes with arbitrary row / batch strides (bytes): box = one 128-byte K block x box_rows rows, 128B
// swizzle (the fp8 row GEMM's operands)
int make_fp8_rows_tmap(CUtensorMap* out, const void* ptr, long long K, long long rows, long long batches, long long row_stride,
                       long long batch_stride, int box_rows) {
  ViewSpec v{ptr, {K, rows, batches, 1}, {row_stride, batches > 1 ? batch_stride : 0, 0}, {128, box_rows, 1, 1},
             CU_TENSOR_MAP_DATA_TYPE_UINT8};
  return make_tmap(out, v);
}

// ------------------------------------------------------------------ launch
template <int BLOCK_N, bool A_MN, bool B_MN>
static int launch_gemm(const CUtensorMap& ta, const CUtensorMap& tb, const GemmParams& p, dim3 grid,
                       cudaStream_t stream) {
  using Cfg = GemmCfg<BLOCK_N>;
  static std::once_flag once;
  static cudaError_t attr_err = cudaSuccess;
  std::call_once(once, [] {
    attr_err = cudaFuncSetAttribute(gemm_bf16_kernel<BLOCK_N, A_MN, B_MN>,
                                    cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::kSmemBytes);
  });
  B200_CHECK_CUDA(attr_err);
  B200_CHECK_CUDA(launch_pdl(gemm_bf16_kernel<BLOCK_N, A_MN, B_MN>, dim3(grid), dim3(Cfg::kThreads), Cfg::kSmemBytes, stream, ta, tb, p));
  B200_CHECK_LAUNCH();
  return 0;
}

static void fill_epilogue(GemmParams& p, const b200s_epilogue* e) {
  p.bias = nullptr;
  p.colsum = nullptr;
  p.out2 = {nullptr, 0, 0};
  p.aux = {nullptr, 0, 0};
  p.res1 = {nullptr, 0, 0};
  p.res2 = {nullptr, 0, 0};
  if (!e) return;
  p.bias = e->bias;
  p.colsum = e->colsum;
  if (e->colsum) p.flags |= EPI_COLSUM;
  if (e->gelu) {
    p.flags |= EPI_GELU;
    if (e->gelu == 2) p.flags |= EPI_GELU_STORE_GRAD;
    p.out2 = {e->out_pre, e->pre_bs, e->pre_ld};
  }
  if (e->dgelu) {
    p.flags |= EPI_DGELU;
    if (e->dgelu == 2) p.flags |= EPI_AUX_IS_GRAD;
    p.aux = {const_cast<void*>(e->gelu_aux), e->aux_bs, e->aux_ld};
  }
  p.res1 = {const_cast<void*>(e->res1), e->res1_bs, e->res1_ld};
  p.res2 = {const_cast<void*>(e->res2), e->res2_bs, e->res2_ld};
}

static int check_epilogue(const b200s_epilogue* e) {
  if (!e) return 0;
  B200_CHECK_ARG(!(e->dgelu && !e->gelu_aux), "epilogue: dgelu requires gelu_aux");
  B200_CHECK_ARG(!(e->gelu && e->dgelu), "epilogue: gelu and dgelu are exclusive");
  return 0;
}

}  // namespace b200

using namespace b200;

extern "C" {

int b200s_version(void) { return 100; }
long long b200s_launch_count(void) { return b200::g_launch_count; }
const char* b200s_last_error(void) { return b200::last_error_buf(); }

// zero `bytes` bytes of device memory on the stream (cudaMemsetAsync: the copy engine's fill, no SM kernel): the per-step reset of
// the flat gradient buffer the backward kernels accumulate into
int b200s_memset_zero(void* p, unsigned long long bytes, b200s_stream stream) {
  B200_CHECK_ARG(p != nullptr || bytes == 0, "memset_zero: null pointer");
  if (bytes == 0) return 0;
  B200_CHECK_CUDA(cudaMemsetAsync(p, 0, static_cast<size_t>(bytes), static_cast<cudaStream_t>(stream)));
  return 0;
}

int b200s_check_device(void) {
  int dev = 0;
  B200_CHECK_CUDA(cudaGetDevice(&dev));
  int major = 0, minor = 0;
  B200_CHECK_CUDA(cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, dev));
  B200_CHECK_CUDA(cudaDeviceGetAttribute(&minor, cudaDevAttrComputeCapabilityMinor, dev));
  B200_CHECK_ARG(major == 9 && minor == 0, "unispeech_b200 needs an sm_90 device (H100); found sm_%d%d", major, minor);
  return 0;
}

static int gemm_rows_impl(const void* a, long long a_bs, long long a_rs, int rows, int batches, int K, const void* w, int N,
                          void* out, long long out_bs, long long out_ld, const b200s_epilogue* epi, const int* m_valid,
                          b200s_stream stream) {
  B200_CHECK_ARG(a && w && out, "gemm_rows: null pointer");
  B200_CHECK_ARG(rows > 0 && batches > 0 && K > 0 && N > 0, "gemm_rows: bad sizes");
  B200_CHECK_ARG(K % 64 == 0, "gemm_rows: K=%d must be a multiple of 64", K);
  B200_CHECK_ARG(N % 8 == 0, "gemm_rows: N=%d must be a multiple of 8", N);
  if (check_epilogue(epi)) return -1;
  cudaStream_t st = static_cast<cudaStream_t>(stream);

  CUtensorMap ta, tb;
  ViewSpec va{a, {K, rows, batches, 1}, {a_rs, batches > 1 ? a_bs : 0, 0}, {64, 128, 1, 1}};
  if (batches == 1) va.strides[1] = 0;
  if (make_tmap(&ta, va)) return -3;

  GemmParams p;
  memset(&p, 0, sizeof(p));
  fill_epilogue(p, epi);
  p.out = {out, out_bs, out_ld};
  p.m_rows = rows;
  p.m_tile_stride = 128;
  p.m_tile_valid = 128;
  p.m_tiles_per_batch = ceil_div(rows, 128);
  p.m_tiles = p.m_tiles_per_batch * batches;
  p.n_total = N;
  p.k_blocks = K / 64;
  // ragged batch: tiles beyond a batch's valid rows are zero-filled instead of computed
  p.m_valid = m_valid;

  if (N >= 256 && m_valid == nullptr) {
    // persistent 128 x 256 kernel.  Narrower outputs keep the 128 x 64 / 128 x 128 tiles, which compute no padded columns;
    // ragged batches keep them too: their dead tiles end a CTA at once and the hardware hands its SM the next live tile, which
    // a static persistent walk cannot match (measured ~1 ms per WavLM-Large ragged step slower even with live tiles first)
    ViewSpec vb{w, {K, N, 1, 1}, {K, 0, 0}, {64, 256, 1, 1}};
    if (make_tmap(&tb, vb)) return -3;
    static std::once_flag once;
    static cudaError_t attr_err = cudaSuccess;
    std::call_once(once, [] {
      attr_err = cudaFuncSetAttribute(gemm_ws_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, WsCfg::kSmemBytes);
    });
    B200_CHECK_CUDA(attr_err);
    const int tiles = p.m_tiles * ceil_div(N, 256);
    B200_CHECK_CUDA(launch_pdl(gemm_ws_kernel, dim3(std::min(tiles, sm_count())), dim3(WsCfg::kThreads), WsCfg::kSmemBytes, st,
                               ta, tb, p));
    B200_CHECK_LAUNCH();
    return 0;
  }

  const int block_n = (N >= 128) ? 128 : 64;
  ViewSpec vb{w, {K, N, 1, 1}, {K, 0, 0}, {64, block_n, 1, 1}};
  if (make_tmap(&tb, vb)) return -3;

  p.n_out_stride = block_n;
  p.n_tile_valid = block_n;
  p.k_blocks_per_batch = 0;
  p.k_blocks_per_split = p.k_blocks;
  // A coords: (k0, m0, mb, 0)   B coords: (k0, n_tile*block_n, 0, 0)
  p.ca[0][4] = 1; p.ca[1][1] = 1; p.ca[2][2] = 1;
  p.cb[0][4] = 1; p.cb[1][3] = block_n;
  dim3 grid(ceil_div(N, block_n), p.m_tiles_per_batch * batches, 1);
  B200_CHECK_ARG(grid.y <= 65535, "gemm_rows: too many M tiles (%u)", grid.y);
  return block_n == 128 ? launch_gemm<128, false, false>(ta, tb, p, grid, st)
                        : launch_gemm<64, false, false>(ta, tb, p, grid, st);
}

/* Deprecated (see the header): range check only. */
int b200s_reserve_sms(int sms) {
  B200_CHECK_ARG(sms >= 0 && sms < sm_count(), "reserve_sms: %d out of range", sms);
  return 0;
}

int b200s_gemm_rows(const void* a, long long a_bs, long long a_rs, int rows, int batches, int K, const void* w, int N,
                    void* out, long long out_bs, long long out_ld, const b200s_epilogue* epi, b200s_stream stream) {
  return gemm_rows_impl(a, a_bs, a_rs, rows, batches, K, w, N, out, out_bs, out_ld, epi, nullptr, stream);
}

int b200s_gemm_rows_ragged(const void* a, long long a_bs, long long a_rs, int rows, int batches, int K, const void* w, int N,
                           void* out, long long out_bs, long long out_ld, const b200s_epilogue* epi, const int* m_valid,
                           b200s_stream stream) {
  return gemm_rows_impl(a, a_bs, a_rs, rows, batches, K, w, N, out, out_bs, out_ld, epi, m_valid, stream);
}

static int gemm_wgrad_impl(const void* y, long long y_bs, long long y_rs, const void* x, long long x_bs, long long x_rs,
                           int rows, int batches, int N, int K, float* dw, long long dw_ld, const int* k_valid,
                           b200s_stream stream) {
  B200_CHECK_ARG(y && x && dw, "gemm_wgrad: null pointer");
  B200_CHECK_ARG(rows > 0 && batches > 0 && K > 0 && N > 0, "gemm_wgrad: bad sizes");
  B200_CHECK_ARG(N % 8 == 0 && K % 8 == 0, "gemm_wgrad: N=%d, K=%d must be multiples of 8", N, K);
  cudaStream_t st = static_cast<cudaStream_t>(stream);

  CUtensorMap ta, tb;
  ViewSpec va{y, {N, rows, batches, 1}, {y_rs, batches > 1 ? y_bs : 0, 0}, {64, 64, 1, 1}};
  if (make_tmap(&ta, va)) return -3;
  ViewSpec vb{x, {K, rows, batches, 1}, {x_rs, batches > 1 ? x_bs : 0, 0}, {64, 64, 1, 1}};
  if (make_tmap(&tb, vb)) return -3;

  GemmParams p;
  memset(&p, 0, sizeof(p));
  p.m_rows = N;
  p.m_tile_stride = 128;
  p.m_tile_valid = 128;
  p.m_tiles_per_batch = ceil_div(N, 128);
  p.n_total = K;
  p.k_blocks_per_batch = ceil_div(rows, 64);
  p.k_blocks = p.k_blocks_per_batch * batches;
  p.flags = EPI_OUT_F32 | EPI_ATOMIC;
  fill_epilogue(p, nullptr);
  p.out = {dw, 0, dw_ld};
  // ragged batch: row blocks beyond a batch's valid rows are neither loaded nor multiplied
  p.k_valid = k_valid;

  if (K >= 256) {
    // persistent 128 x 256 stream-K kernel.  Narrower outputs keep the 128 x 64 tiles, which compute no padded columns.
    p.m_tiles = p.m_tiles_per_batch;
    static std::once_flag once;
    static cudaError_t attr_err = cudaSuccess;
    std::call_once(once, [] {
      attr_err = cudaFuncSetAttribute(gemm_ws_wgrad_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, WsCfg::kSmemBytes);
    });
    B200_CHECK_CUDA(attr_err);
    const long long work = static_cast<long long>(p.m_tiles) * ceil_div(K, 256) * p.k_blocks;
    B200_CHECK_CUDA(launch_pdl(gemm_ws_wgrad_kernel, dim3(static_cast<unsigned>(std::min<long long>(work, sm_count()))),
                               dim3(WsCfg::kThreads), WsCfg::kSmemBytes, st, ta, tb, p));
    B200_CHECK_LAUNCH();
    return 0;
  }

  const int block_n = 64;
  p.n_out_stride = block_n;
  p.n_tile_valid = block_n;
  const int tiles = p.m_tiles_per_batch * ceil_div(K, block_n);
  int splits = ceil_div(2 * sm_count(), tiles);
  if (splits > p.k_blocks) splits = p.k_blocks;
  if (splits < 1) splits = 1;
  p.k_blocks_per_split = ceil_div(p.k_blocks, splits);
  splits = ceil_div(p.k_blocks, p.k_blocks_per_split);
  // A coords: (m0 + sub, k0, kbatch, 0)   B coords: (n_tile*block_n + sub, k0, kbatch, 0)
  p.ca[0][1] = 1; p.ca[0][7] = 1; p.ca[1][4] = 1; p.ca[2][5] = 1;
  p.cb[0][3] = block_n; p.cb[0][7] = 1; p.cb[1][4] = 1; p.cb[2][5] = 1;
  dim3 grid(ceil_div(K, block_n), p.m_tiles_per_batch, splits);
  return launch_gemm<64, true, true>(ta, tb, p, grid, st);
}

int b200s_gemm_wgrad(const void* y, long long y_bs, long long y_rs, const void* x, long long x_bs, long long x_rs,
                     int rows, int batches, int N, int K, float* dw, long long dw_ld, b200s_stream stream) {
  return gemm_wgrad_impl(y, y_bs, y_rs, x, x_bs, x_rs, rows, batches, N, K, dw, dw_ld, nullptr, stream);
}

int b200s_gemm_wgrad_ragged(const void* y, long long y_bs, long long y_rs, const void* x, long long x_bs, long long x_rs,
                            int rows, int batches, int N, int K, float* dw, long long dw_ld, const int* k_valid,
                            b200s_stream stream) {
  return gemm_wgrad_impl(y, y_bs, y_rs, x, x_bs, x_rs, rows, batches, N, K, dw, dw_ld, k_valid, stream);
}

int b200s_posconv_gemm(const void* xpad, long long xpad_bs, int T, int B, int D, int G, int taps, const void* wp,
                       void* out, long long out_bs, long long out_ld, const b200s_epilogue* epi,
                       b200s_stream stream) {
  B200_CHECK_ARG(xpad && wp && out, "posconv_gemm: null pointer");
  B200_CHECK_ARG(D % G == 0, "posconv_gemm: D %% G != 0");
  const int Cg = D / G;
  B200_CHECK_ARG(Cg <= 128 && Cg % 8 == 0, "posconv_gemm: channels per group %d must be <=128 and a multiple of 8", Cg);
  B200_CHECK_ARG(D % 8 == 0, "posconv_gemm: D must be a multiple of 8");
  B200_CHECK_ARG(taps >= 1, "posconv_gemm: taps=%d must be positive", taps);
  const int KB = Cg <= 64 ? 1 : 2;  // 64-channel blocks of the padded group width Cgp
  B200_CHECK_ARG(KB == 1 || taps <= 129, "posconv_gemm: %d channels per group needs taps <= 129 (got %d)", Cg, taps);
  if (check_epilogue(epi)) return -1;

  CUtensorMap ta, tb;
  ViewSpec vb{wp, {taps * 64LL * KB, G * 64LL * KB, 1, 1}, {taps * 64LL * KB, 0, 0}, {64, 64, 1, 1}};
  if (make_tmap(&tb, vb)) return -3;

  GemmParams p;
  memset(&p, 0, sizeof(p));
  p.m_rows = T;
  p.m_tile_stride = 128;
  p.m_tile_valid = 128;
  p.m_tiles_per_batch = ceil_div(T, 128);
  p.n_total = D;
  p.n_out_stride = Cg;
  p.n_tile_valid = Cg;
  p.k_blocks = taps;
  p.k_blocks_per_batch = 0;
  p.k_blocks_per_split = taps;
  p.flags = 0;
  fill_epilogue(p, epi);
  p.out = {out, out_bs, out_ld};
  dim3 grid(G * KB, p.m_tiles_per_batch * B, 1);
  cudaStream_t st = static_cast<cudaStream_t>(stream);

  if (taps <= 129) {
    // windowed kernel: the A operand (256 input rows of this group's channels) is loaded once per tile, every tap reads it
    // shifted by one row; rows past T + taps - 1 (end of this utterance's zero padding) are zero-filled by the tensor map
    ViewSpec vw{xpad, {D, T + taps - 1, B, 1}, {D, B > 1 ? xpad_bs : 0, 0}, {64, 256, 1, 1}};
    if (make_tmap(&ta, vw)) return -3;
    static std::once_flag once;
    static cudaError_t attr_err = cudaSuccess;
    std::call_once(once, [] {
      attr_err = cudaFuncSetAttribute(posconv_window_kernel<1>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                      PosconvCfg<1>::kSmemBytes);
      if (attr_err == cudaSuccess)
        attr_err = cudaFuncSetAttribute(posconv_window_kernel<2>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                        PosconvCfg<2>::kSmemBytes);
    });
    B200_CHECK_CUDA(attr_err);
    if (KB == 1)
      B200_CHECK_CUDA(launch_pdl(posconv_window_kernel<1>, grid, dim3(PosconvCfg<1>::kThreads), PosconvCfg<1>::kSmemBytes, st, ta,
                                 tb, p, taps, Cg));
    else
      B200_CHECK_CUDA(launch_pdl(posconv_window_kernel<2>, grid, dim3(PosconvCfg<2>::kThreads), PosconvCfg<2>::kSmemBytes, st, ta,
                                 tb, p, taps, Cg));
    B200_CHECK_LAUNCH();
    return 0;
  }
  // box-per-tap formulation (any tap count)
  ViewSpec va{xpad, {D, taps, T, B}, {D, D, xpad_bs}, {64, 1, 128, 1}};
  if (make_tmap(&ta, va)) return -3;
  // A coords: (g*Cg, kb, m0, mb)   B coords: (kb*64, g*64, 0, 0)
  p.ca[0][3] = Cg; p.ca[1][6] = 1; p.ca[2][1] = 1; p.ca[3][2] = 1;
  p.cb[0][4] = 1; p.cb[1][3] = 64;
  return launch_gemm<64, false, false>(ta, tb, p, grid, st);
}

int b200s_posconv_wgrad(const void* dy, long long dy_bs, long long dy_rs, const void* xpad, long long xpad_bs, int T,
                        int B, int D, int G, int taps, float* dwp, b200s_stream stream) {
  B200_CHECK_ARG(dy && xpad && dwp, "posconv_wgrad: null pointer");
  B200_CHECK_ARG(D % G == 0, "posconv_wgrad: D %% G != 0");
  const int Cg = D / G;
  B200_CHECK_ARG(Cg <= 128 && Cg % 8 == 0, "posconv_wgrad: channels per group %d must be <=128 and a multiple of 8", Cg);
  const int Cgp = Cg <= 64 ? 64 : 128;

  CUtensorMap ta;
  ViewSpec va{dy, {D, T, B, 1}, {dy_rs, B > 1 ? dy_bs : 0, 0}, {64, 64, 1, 1}};
  if (make_tmap(&ta, va)) return -3;
  // one launch per 64 input channels of the group: launch h reads xpad from channel 64 h of each group on (a view whose
  // channels past D are zero-filled) and writes columns 64 h .. of each tap's Cgp-wide block of dwp
  for (int h = 0; h * 64 < Cg; ++h) {
    CUtensorMap tb;
    ViewSpec vb{static_cast<const __nv_bfloat16*>(xpad) + 64 * h, {D - 64 * h, taps, T, B}, {D, D, xpad_bs}, {64, 1, 64, 1}};
    if (make_tmap(&tb, vb)) return -3;

    GemmParams p;
    memset(&p, 0, sizeof(p));
    p.m_rows = D;
    p.m_tile_stride = Cg;
    p.m_tile_valid = Cg;
    p.m_tiles_per_batch = G;
    p.n_total = taps * Cgp;
    p.n_out_stride = Cgp;
    p.n_tile_valid = h == 0 ? 64 : Cg - 64 * h;  // (columns past Cg are never read)
    p.k_blocks_per_batch = ceil_div(T, 64);
    p.k_blocks = p.k_blocks_per_batch * B;
    p.k_blocks_per_split = p.k_blocks;
    // A coords: (m0 + sub, k0, kbatch, 0)   B coords: (m0, tap = n_tile, k0, kbatch)
    p.ca[0][1] = 1; p.ca[0][7] = 1; p.ca[1][4] = 1; p.ca[2][5] = 1;
    p.cb[0][1] = 1; p.cb[1][3] = 1; p.cb[2][4] = 1; p.cb[3][5] = 1;
    p.flags = EPI_OUT_F32 | EPI_ATOMIC;
    fill_epilogue(p, nullptr);
    p.out = {dwp + 64 * h, 0, taps * static_cast<long long>(Cgp)};
    dim3 grid(taps, G, 1);
    if (const int rc = launch_gemm<64, true, true>(ta, tb, p, grid, static_cast<cudaStream_t>(stream))) return rc;
  }
  return 0;
}

}  // extern "C"
