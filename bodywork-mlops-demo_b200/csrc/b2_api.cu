// b2_api.cu -- the C-ABI of libb2gram.so (declared in include/b2gram.h): context, caller-buffer
// helpers, dispatch between the tensor-core and CUDA-core Gram kernels, host-streamed accumulation
// (pinned ring -> HBM staging, copy/compute overlap), NCCL all-reduce of the statistic, timing.
#include <dlfcn.h>
#include <math.h>
#include <stdarg.h>
#include <stdlib.h>

#include <new>
#include <thread>
#include <vector>

#include "b2_internal.cuh"
#include "b2_xchg.cuh"

namespace b2 {

static thread_local char g_err[768] = "";

void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}

namespace {

// ---- NCCL through dlopen: no link-time dependency, the library loads on CPU-only boxes ------------
struct NcclUid { char internal[128]; };
struct NcclApi {
  void* lib = nullptr;
  int (*GetUniqueId)(NcclUid*) = nullptr;
  int (*CommInitRank)(void**, int, NcclUid, int) = nullptr;
  int (*CommDestroy)(void*) = nullptr;
  int (*AllReduce)(const void*, void*, size_t, int, int, void*, cudaStream_t) = nullptr;
  const char* (*GetErrorString)(int) = nullptr;
};
constexpr int kNcclFloat64 = 8, kNcclSum = 0, kNcclMax = 2;

NcclApi* nccl() {
  static NcclApi api;
  static bool tried = false;
  if (!tried) {
    tried = true;
    const char* names[] = {"libnccl.so.2", "libnccl.so"};
    for (const char* nm : names) {
      api.lib = dlopen(nm, RTLD_NOW | RTLD_GLOBAL);
      if (api.lib) break;
    }
    if (api.lib) {
      api.GetUniqueId = reinterpret_cast<int (*)(NcclUid*)>(dlsym(api.lib, "ncclGetUniqueId"));
      api.CommInitRank = reinterpret_cast<int (*)(void**, int, NcclUid, int)>(dlsym(api.lib, "ncclCommInitRank"));
      api.CommDestroy = reinterpret_cast<int (*)(void*)>(dlsym(api.lib, "ncclCommDestroy"));
      api.AllReduce = reinterpret_cast<int (*)(const void*, void*, size_t, int, int, void*, cudaStream_t)>(
          dlsym(api.lib, "ncclAllReduce"));
      api.GetErrorString = reinterpret_cast<const char* (*)(int)>(dlsym(api.lib, "ncclGetErrorString"));
    }
  }
  if (!api.lib || !api.GetUniqueId || !api.CommInitRank || !api.AllReduce) return nullptr;
  return &api;
}

#define B2_NCCL(api, call)                                                                     \
  do {                                                                                         \
    int r_ = (call);                                                                           \
    if (r_ != 0) {                                                                             \
      set_error("%s failed: %s", #call, (api)->GetErrorString ? (api)->GetErrorString(r_) : "?"); \
      return B2_E_COMM;                                                                        \
    }                                                                                          \
  } while (0)

int use_device(b2_ctx* ctx) {
  if (ctx == nullptr) {
    set_error("null context");
    return B2_E_ARG;
  }
  B2_CUDA(cudaSetDevice(ctx->device));
  return B2_OK;
}

int check_shape(int x_dtype, int64_t n, int d, int64_t ldx, int mem_kind) {
  if (x_dtype != B2_F32 && x_dtype != B2_BF16) { set_error("x_dtype must be B2_F32 or B2_BF16"); return B2_E_ARG; }
  if (d < 1 || d > kMaxD) { set_error("d=%d out of range [1,%d]", d, kMaxD); return B2_E_ARG; }
  if (n < 0) { set_error("n_rows < 0"); return B2_E_ARG; }
  if (ldx < d) { set_error("ldx=%lld < d=%d", (long long)ldx, d); return B2_E_ARG; }
  if (mem_kind != B2_MEM_DEVICE && mem_kind != B2_MEM_HOST) { set_error("bad mem_kind %d", mem_kind); return B2_E_ARG; }
  return B2_OK;
}

constexpr int64_t kMaxRowsPerLaunch = (int64_t)1 << 30;   // TMA coordinates / tile counters are int32

// Device-resident rows into S: the one place that picks a Gram kernel.  Blocks of more than kMaxRowsPerLaunch rows
// take several launches.  Per launch, the rows the main kernel's tiling leaves over (packing remainder, partial
// narrow tile; all rows on the SIMT kernel) run first on the exact fp64 kernel, then the main kernel takes the first
// main_rows rows.  Before both, the shift sample of the tensor-core and narrow kernels covers all rows of the launch.
// The first kernel to write S after b2_gram_reset overwrites it.
// scatter_epoch != nullptr (b2_fit): with an attached peer exchange, a final tensor-core launch stores S into the
// peers' exchange slots, and *scatter_epoch is that exchange's number (0: none).  *tc_last: the final launch was
// tensor-core.
int gram_dispatch(b2_ctx* ctx, const void* X, int x_dtype, const float* y, int64_t n, int d, int64_t ldx,
                  const uint8_t* mask, int keep, bool* tc_last = nullptr, unsigned int* scatter_epoch = nullptr) {
  const int es = x_dtype == B2_F32 ? 4 : 2;
  for (int64_t r0 = 0; r0 < n; r0 += kMaxRowsPerLaunch) {
    const int64_t rows = n - r0 < kMaxRowsPerLaunch ? n - r0 : kMaxRowsPerLaunch;
    const char* Xb = static_cast<const char*>(X) + (size_t)r0 * ldx * es;
    const float* yb = y + r0;
    const uint8_t* mb = mask != nullptr ? mask + r0 : nullptr;
    const bool tc_ok = gram_tc_supported(Xb, x_dtype, yb, rows, d, ldx, mb);
    const bool nw_ok = gram_narrow_supported(Xb, x_dtype, yb, rows, d, ldx, mb);
    int mode = ctx->kernel_mode;
    if (mode == B2_KERNEL_TCGEN05 && !tc_ok) {
      set_error("tensor-core path needs d%%4==0 (fp32) / d%%8==0 (bf16), 16-byte aligned X/y/mask/row pitch, n>=32");
      return B2_E_UNSUPPORTED;
    }
    if (mode == B2_KERNEL_NARROW && !nw_ok) {
      set_error("narrow path needs d<=16, contiguous rows (ldx==d) and 16-byte aligned X/y/mask");
      return B2_E_UNSUPPORTED;
    }
    if (mode == B2_KERNEL_AUTO) {
      // narrow rows stream through the CUDA-core pipeline (HBM-bound); wide rows go to the tensor core;
      // tiny tranches (the reference's 1 440-row day) and odd layouts stay on the exact fp64 kernel
      if (nw_ok && rows >= 4096) mode = B2_KERNEL_NARROW;
      else mode = (tc_ok && rows >= 2048) ? B2_KERNEL_TCGEN05 : B2_KERNEL_SIMT;
    }
    const int64_t main_rows = mode == B2_KERNEL_NARROW ? gram_narrow_main_rows(rows, d)
                            : mode == B2_KERNEL_TCGEN05 ? gram_tc_main_rows(rows, d, ldx, nullptr) : 0;
    if (main_rows > 0)
      if (int r = launch_gram_shift(ctx, Xb, x_dtype, yb, rows, d, ldx)) return r;
    if (main_rows < rows) {
      if (int r = launch_gram_simt(ctx, Xb + (size_t)main_rows * ldx * es, x_dtype, yb + main_rows, rows - main_rows, d,
                                   ldx, mb != nullptr ? mb + main_rows : nullptr, keep, ctx->s_zero_pending))
        return r;
      ctx->s_zero_pending = false;
    }
    const bool last = r0 + rows == n;
    if (main_rows > 0 && mode == B2_KERNEL_NARROW) {
      if (int r = launch_gram_narrow(ctx, Xb, x_dtype, yb, rows, d, mb, keep, ctx->s_zero_pending)) return r;
      ctx->s_zero_pending = false;
    } else if (main_rows > 0) {
      const unsigned int epoch =
          last && scatter_epoch != nullptr && ctx->n_ranks > 1 && ctx->p2p_ready ? ++ctx->xchg_epoch : 0u;
      if (int r = launch_gram_tc(ctx, Xb, x_dtype, yb, rows, d, ldx, mb, keep, ctx->s_zero_pending, epoch)) return r;
      ctx->s_zero_pending = false;
      if (scatter_epoch != nullptr) *scatter_epoch = epoch;
    }
    if (last && tc_last != nullptr) *tc_last = mode == B2_KERNEL_TCGEN05;
  }
  return B2_OK;
}

int ensure_staging(b2_ctx* ctx) {
  if (ctx->stage_x[0] != nullptr) return B2_OK;
  ctx->stage_rows = 1 << 18;                                  // 262 144 rows per block (134 MB at 128 x fp32)
  ctx->stage_bytes_x = (size_t)ctx->stage_rows * kMaxD * 4;
  for (int b = 0; b < 2; ++b) {
    B2_CUDA(cudaMalloc(&ctx->stage_x[b], ctx->stage_bytes_x));
    B2_CUDA(cudaMalloc(reinterpret_cast<void**>(&ctx->stage_y[b]), (size_t)ctx->stage_rows * 4));
    B2_CUDA(cudaMalloc(reinterpret_cast<void**>(&ctx->stage_m[b]), (size_t)ctx->stage_rows));
    B2_CUDA(cudaEventCreateWithFlags(&ctx->ev_copied[b], cudaEventDisableTiming));
    B2_CUDA(cudaEventCreateWithFlags(&ctx->ev_consumed[b], cudaEventDisableTiming));
  }
  return B2_OK;
}

// Is a host pointer page-locked (cudaHostAlloc / cudaHostRegister)?  Pageable rows -- what numpy / pandas hand over --
// cannot be DMA'ed directly: the driver bounces them through one internal staging buffer on one thread (~11 GB/s
// measured here).  They take the library's own bounce ring instead: several host threads copy the next block into a
// pinned buffer while the previous block is on the wire.
bool host_pointer_is_pinned(const void* p) {
  cudaPointerAttributes attr;
  if (cudaPointerGetAttributes(&attr, p) != cudaSuccess) { cudaGetLastError(); return false; }
  return attr.type == cudaMemoryTypeHost || attr.type == cudaMemoryTypeManaged;
}

int ensure_bounce(b2_ctx* ctx) {
  if (ctx->bounce[0] != nullptr) return B2_OK;
  for (int b = 0; b < 2; ++b) {
    B2_CUDA(cudaHostAlloc(&ctx->bounce[b], ctx->stage_bytes_x, cudaHostAllocDefault));
    B2_CUDA(cudaEventCreateWithFlags(&ctx->ev_bounce[b], cudaEventDisableTiming));
  }
  return B2_OK;
}

static int copy_threads() {
  static const int nt_cfg = []() {
    const char* e = getenv("B2_COPY_THREADS");
    if (e != nullptr && atoi(e) > 0) return atoi(e) > 64 ? 64 : atoi(e);
    const unsigned hw = std::thread::hardware_concurrency();
    const int half = (int)(hw / 2);
    return half < 4 ? 4 : (half > 16 ? 16 : half);
  }();
  return nt_cfg;
}

void parallel_copy_rows(char* dst, const char* src, int64_t rows, size_t row_bytes, size_t src_pitch) {
  // copy threads: half the hardware threads, at most 16;
  // B2_COPY_THREADS overrides
  int nt = copy_threads();
  if ((size_t)rows * row_bytes < ((size_t)8 << 20)) nt = 1;
  auto work = [=](int t) {
    const int64_t lo = rows * t / nt, hi = rows * (t + 1) / nt;
    if (src_pitch == row_bytes) {
      memcpy(dst + (size_t)lo * row_bytes, src + (size_t)lo * src_pitch, (size_t)(hi - lo) * row_bytes);
    } else {
      for (int64_t r = lo; r < hi; ++r) memcpy(dst + (size_t)r * row_bytes, src + (size_t)r * src_pitch, row_bytes);
    }
  };
  if (nt == 1) { work(0); return; }
  std::vector<std::thread> pool;
  pool.reserve(nt - 1);
  for (int t = 1; t < nt; ++t) pool.emplace_back(work, t);
  work(0);
  for (auto& th : pool) th.join();
}

// gather + convert `rows` rows of d strided host columns into a row-major fp32 block (b2_upload_columns)
template <typename T>
static void pack_rows(float* dst, const void* const* cols, const int64_t* strides, int64_t r0, int64_t rows, int d) {
  constexpr int kRowsPerTile = 64, kColsPerPass = 16;
  for (int64_t t0 = 0; t0 < rows; t0 += kRowsPerTile) {
    const int64_t tr = rows - t0 < kRowsPerTile ? rows - t0 : kRowsPerTile;
    for (int j0 = 0; j0 < d; j0 += kColsPerPass) {
      const int jc = d - j0 < kColsPerPass ? d - j0 : kColsPerPass;
      const char* src[kColsPerPass];
      int64_t st[kColsPerPass];
      for (int j = 0; j < jc; ++j) { st[j] = strides[j0 + j]; src[j] = static_cast<const char*>(cols[j0 + j]) + (r0 + t0) * st[j]; }
      for (int64_t r = 0; r < tr; ++r) {
        float* out = dst + (size_t)(t0 + r) * d + j0;
        for (int j = 0; j < jc; ++j) out[j] = (float)*reinterpret_cast<const T*>(src[j] + r * st[j]);
      }
    }
  }
}

// copy rows [r0, r0+rows) of a host matrix into a compact (ldx == d) staging block
int stage_rows_h2d(b2_ctx* ctx, int buf, const void* X, int es, const float* y, const uint8_t* mask, int64_t r0,
                   int64_t rows, int d, int64_t ldx, bool pinned) {
  const char* src = static_cast<const char*>(X) + (size_t)r0 * ldx * es;
  if (!pinned) {
    if (int r = ensure_bounce(ctx)) return r;
    B2_CUDA(cudaEventSynchronize(ctx->ev_bounce[buf]));                 // the H2D that last read this bounce block is done
    parallel_copy_rows(static_cast<char*>(ctx->bounce[buf]), src, rows, (size_t)d * es, (size_t)ldx * es);
    B2_CUDA(cudaMemcpyAsync(ctx->stage_x[buf], ctx->bounce[buf], (size_t)rows * d * es, cudaMemcpyHostToDevice, ctx->copy_stream));
    B2_CUDA(cudaEventRecord(ctx->ev_bounce[buf], ctx->copy_stream));
  } else if (ldx == d) {
    B2_CUDA(cudaMemcpyAsync(ctx->stage_x[buf], src, (size_t)rows * d * es, cudaMemcpyHostToDevice, ctx->copy_stream));
  } else {
    B2_CUDA(cudaMemcpy2DAsync(ctx->stage_x[buf], (size_t)d * es, src, (size_t)ldx * es, (size_t)d * es, rows,
                              cudaMemcpyHostToDevice, ctx->copy_stream));
  }
  if (y != nullptr)
    B2_CUDA(cudaMemcpyAsync(ctx->stage_y[buf], y + r0, (size_t)rows * 4, cudaMemcpyHostToDevice, ctx->copy_stream));
  if (mask != nullptr)
    B2_CUDA(cudaMemcpyAsync(ctx->stage_m[buf], mask + r0, (size_t)rows, cudaMemcpyHostToDevice, ctx->copy_stream));
  return B2_OK;
}

// Host rows through the two-deep HBM staging ring, in blocks of blk_rows: stage(buf, r0, rows) enqueues the copies of
// one block into staging buffer buf on copy_stream, consume(buf, r0, rows) the work that reads it on stream; copies
// overlap the work on the other buffer.  The caller may reuse its host buffers on return -- also when a block failed.
template <typename Stage, typename Consume>
int stream_host_blocks(b2_ctx* ctx, int64_t n_rows, int64_t blk_rows, Stage stage, Consume consume) {
  auto block = [&](int buf, int64_t r0, int64_t rows) -> int {
    // work of this call -- or of an EARLIER call that returned without a stream sync -- may still read this buffer
    if (ctx->ev_consumed_valid[buf]) B2_CUDA(cudaStreamWaitEvent(ctx->copy_stream, ctx->ev_consumed[buf], 0));
    if (int r = stage(buf, r0, rows)) return r;
    B2_CUDA(cudaEventRecord(ctx->ev_copied[buf], ctx->copy_stream));
    B2_CUDA(cudaStreamWaitEvent(ctx->stream, ctx->ev_copied[buf], 0));
    if (int r = consume(buf, r0, rows)) return r;
    B2_CUDA(cudaEventRecord(ctx->ev_consumed[buf], ctx->stream));
    ctx->ev_consumed_valid[buf] = true;
    return B2_OK;
  };
  int rc = B2_OK;
  int64_t blk = 0;
  for (int64_t r0 = 0; r0 < n_rows && rc == B2_OK; r0 += blk_rows, ++blk)
    rc = block((int)(blk & 1), r0, n_rows - r0 < blk_rows ? n_rows - r0 : blk_rows);
  const cudaError_t drained = cudaStreamSynchronize(ctx->copy_stream);
  if (rc != B2_OK) return rc;
  B2_CUDA(drained);
  return B2_OK;
}

// The row-output blocks grown to block_bytes each (their contents are not kept)
int ensure_row_out(b2_ctx* ctx, size_t block_bytes) {
  if (ctx->row_out_bytes >= block_bytes) return B2_OK;
  if (ctx->row_out[0] != nullptr) B2_CUDA(cudaStreamSynchronize(ctx->stream));   // an earlier call's copies may still read them
  for (int b = 0; b < 2; ++b) {
    if (ctx->row_out[b] != nullptr) cudaFree(ctx->row_out[b]);
    ctx->row_out[b] = nullptr;
  }
  ctx->row_out_bytes = 0;
  for (int b = 0; b < 2; ++b)
    if (cudaMalloc(reinterpret_cast<void**>(&ctx->row_out[b]), block_bytes) != cudaSuccess) {
      cudaGetLastError();
      set_error("out of device memory for the staging blocks of the per-row outputs");
      return B2_E_CUDA;
    }
  ctx->row_out_bytes = block_bytes;
  return B2_OK;
}

// A per-row output of a row pass: the caller's destination (device memory for device rows, host memory for host rows,
// null: not wanted) and its bytes per row.
struct RowOut {
  void* dst = nullptr;
  size_t row_bytes = 0;
};

// One pass over the rows [0, n_rows) of a call, wherever they live: launch(span, out0, out1, out2) enqueues the pass over
// the rows of `span` and writes the per-row outputs to out0 / out1 / out2 (null when not wanted).
// Device rows: one launch on the caller's pointers.  Host rows: one launch per block of the staging ring, its outputs
// written to the row-output blocks and copied back behind it; with outputs, the stream is synchronised before the
// return, so the caller may reuse every host buffer -- also when a block failed.  Zero rows: one launch on zero rows.
// max_blk_rows > 0 caps the rows of a host block below the staging ring's (wide per-row outputs).
template <typename Launch>
int row_pass(b2_ctx* ctx, const void* X, int x_dtype, const float* y, int64_t n_rows, int d, int64_t ldx, int mem_kind,
             const uint8_t* mask, Launch&& launch, RowOut out0 = {}, RowOut out1 = {}, RowOut out2 = {},
             int64_t max_blk_rows = 0) {
  if (mem_kind == B2_MEM_DEVICE) return launch(RowSpan{X, y, mask, ldx, 0, n_rows, true}, out0.dst, out1.dst, out2.dst);
  if (n_rows == 0) return launch(RowSpan{nullptr, nullptr, nullptr, d, 0, 0, true}, nullptr, nullptr, nullptr);
  if (int r = ensure_staging(ctx)) return r;
  const int64_t blk = max_blk_rows > 0 && max_blk_rows < ctx->stage_rows ? max_blk_rows : ctx->stage_rows;
  RowOut out[3] = {out0, out1, out2};
  size_t out_bytes = 0;
  for (RowOut& o : out) {
    if (o.dst == nullptr) o.row_bytes = 0;
    out_bytes += o.row_bytes;
  }
  if (out_bytes > 0)
    if (int r = ensure_row_out(ctx, (size_t)blk * out_bytes)) return r;
  const int es = x_dtype == B2_F32 ? 4 : 2;
  const bool x_pinned = host_pointer_is_pinned(X);
  const int rc = stream_host_blocks(
      ctx, n_rows, blk,
      [&](int buf, int64_t r0, int64_t rows) {
        return stage_rows_h2d(ctx, buf, X, es, y, mask, r0, rows, d, ldx, x_pinned);
      },
      [&](int buf, int64_t r0, int64_t rows) -> int {
        char* const block = ctx->row_out[buf];   // [blk] of output 0, then of output 1, then of output 2
        char* dev[3] = {out[0].dst != nullptr ? block : nullptr,
                        out[1].dst != nullptr ? block + (size_t)blk * out[0].row_bytes : nullptr,
                        out[2].dst != nullptr ? block + (size_t)blk * (out[0].row_bytes + out[1].row_bytes) : nullptr};
        const RowSpan s{ctx->stage_x[buf], y != nullptr ? ctx->stage_y[buf] : nullptr,
                        mask != nullptr ? ctx->stage_m[buf] : nullptr, d, r0, rows, r0 == 0};
        if (int r = launch(s, dev[0], dev[1], dev[2])) return r;
        for (int k = 0; k < 3; ++k)
          if (out[k].dst != nullptr)
            B2_CUDA(cudaMemcpyAsync(static_cast<char*>(out[k].dst) + (size_t)r0 * out[k].row_bytes, dev[k],
                                    (size_t)rows * out[k].row_bytes, cudaMemcpyDeviceToHost, ctx->stream));
        return B2_OK;
      });
  if (out_bytes == 0) return rc;
  const cudaError_t done = cudaStreamSynchronize(ctx->stream);   // the outputs' copies into the caller's buffers
  if (rc != B2_OK) return rc;
  B2_CUDA(done);
  return B2_OK;
}

// The rows of a call into S through the Gram dispatch (b2_fit's device rows call gram_dispatch themselves, for the
// fused exchange)
int gram_rows(b2_ctx* ctx, const void* X, int x_dtype, const float* y, int64_t n_rows, int d, int64_t ldx, int mem_kind,
              const uint8_t* mask, int keep) {
  return row_pass(ctx, X, x_dtype, y, n_rows, d, ldx, mem_kind, mask, [&](const RowSpan& s, void*, void*, void*) {
    return gram_dispatch(ctx, s.X, x_dtype, s.y, s.rows, d, s.ldx, s.mask, keep);
  });
}

// honours a lazy b2_gram_reset where S is read before any kernel wrote it (exchange, export, solves after zero rows)
int ensure_s_cleared(b2_ctx* ctx) {
  if (ctx->s_zero_pending) {
    B2_CUDA(cudaMemsetAsync(ctx->S, 0, sizeof(double) * kMaxS * kMaxS, ctx->stream));
    ctx->s_zero_pending = false;
  }
  return B2_OK;
}

}  // namespace

}  // namespace b2

using namespace b2;

extern "C" {

int b2_abi_version(void) { return B2_ABI_VERSION; }
const char* b2_last_error(void) { return g_err; }

int b2_device_count(int* n_out) {
  if (n_out == nullptr) { set_error("n_out is null"); return B2_E_ARG; }
  int n = 0;
  cudaError_t e = cudaGetDeviceCount(&n);
  if (e != cudaSuccess) {
    cudaGetLastError();
    *n_out = 0;
    set_error("cudaGetDeviceCount: %s", cudaGetErrorString(e));
    return B2_E_CUDA;
  }
  *n_out = n;
  return B2_OK;
}

// streams, events and device scratch of a fresh context (b2_ctx_create destroys the context if this fails)
static int ctx_allocate(b2_ctx* ctx) {
  B2_CUDA(cudaStreamCreateWithFlags(&ctx->stream, cudaStreamNonBlocking));
  B2_CUDA(cudaStreamCreateWithFlags(&ctx->copy_stream, cudaStreamNonBlocking));
  B2_CUDA(cudaEventCreate(&ctx->ev_t0));
  B2_CUDA(cudaEventCreate(&ctx->ev_t1));
  for (int i = 0; i < kKernelEventPairs; ++i) {
    B2_CUDA(cudaEventCreate(&ctx->ev_k[i][0]));
    B2_CUDA(cudaEventCreate(&ctx->ev_k[i][1]));
  }
  ctx->simt_ctas = ctx->sm_count;
  ctx->score_ctas = ctx->sm_count * 8;
  B2_CUDA(cudaMalloc(reinterpret_cast<void**>(&ctx->S), sizeof(double) * kMaxS * kMaxS));
  B2_CUDA(cudaMalloc(reinterpret_cast<void**>(&ctx->tc_part),
                     sizeof(double) * (size_t)ctx->sm_count * (kTcAccElems + kTcSums)));
  B2_CUDA(cudaMalloc(reinterpret_cast<void**>(&ctx->tc_red), sizeof(double) * (kTcAccElems + 16)));
  B2_CUDA(cudaMalloc(reinterpret_cast<void**>(&ctx->shift), gram_shift_bytes()));
  B2_CUDA(cudaMalloc(reinterpret_cast<void**>(&ctx->simt_part), sizeof(double) * (size_t)ctx->simt_ctas * kMaxS * kMaxS));
  B2_CUDA(cudaMalloc(reinterpret_cast<void**>(&ctx->score_part), sizeof(double) * ((size_t)ctx->score_ctas + 2) * kNStats));
  B2_CUDA(cudaMalloc(reinterpret_cast<void**>(&ctx->coef_dev), sizeof(double) * (kMaxD + 1)));
  B2_CUDA(cudaMalloc(reinterpret_cast<void**>(&ctx->grad_part), sizeof(double) * (size_t)ctx->score_ctas * kGradOut));
  B2_CUDA(cudaMalloc(reinterpret_cast<void**>(&ctx->refine), sizeof(double) * kRfDoubles));
  B2_CUDA(cudaMalloc(reinterpret_cast<void**>(&ctx->loo), sizeof(double) * kLooDoubles));
  B2_CUDA(cudaMalloc(reinterpret_cast<void**>(&ctx->loo_part), sizeof(double) * (size_t)ctx->sm_count * kMaxAlphas));
  B2_CUDA(cudaMalloc(reinterpret_cast<void**>(&ctx->solve_out), sizeof(double) * (2 * kMaxD + 8)));
  B2_CUDA(cudaHostAlloc(reinterpret_cast<void**>(&ctx->solve_host), sizeof(double) * (2 * kMaxD + 8), cudaHostAllocDefault));
  B2_CUDA(cudaMalloc(reinterpret_cast<void**>(&ctx->tc_sync), 64));
  B2_CUDA(cudaMemset(ctx->tc_sync, 0, 64));
  B2_CUDA(cudaHostAlloc(reinterpret_cast<void**>(&ctx->xchg_status_host), 64, cudaHostAllocDefault));
  ctx->xchg_status_host[0] = 0u;
  B2_CUDA(cudaHostAlloc(reinterpret_cast<void**>(&ctx->coef_host), 2 * sizeof(double) * (kMaxD + 1), cudaHostAllocDefault));
  for (int b = 0; b < 2; ++b) B2_CUDA(cudaEventCreateWithFlags(&ctx->ev_coef[b], cudaEventDisableTiming));
  B2_CUDA(cudaMemset(ctx->shift, 0, gram_shift_bytes()));
  B2_CUDA(cudaMemset(ctx->S, 0, sizeof(double) * kMaxS * kMaxS));
  B2_CUDA(cudaMemset(ctx->tc_red, 0, sizeof(double) * (kTcAccElems + 16)));
  return B2_OK;
}

int b2_ctx_create(int device, b2_ctx** out) {
  if (out == nullptr) { set_error("out is null"); return B2_E_ARG; }
  *out = nullptr;
  int n = 0;
  if (b2_device_count(&n) != B2_OK || n == 0) {
    set_error("no usable CUDA device (libb2gram has no CPU fallback)");
    return B2_E_CUDA;
  }
  if (device < 0 || device >= n) { set_error("device %d out of range (0..%d)", device, n - 1); return B2_E_ARG; }
  B2_CUDA(cudaSetDevice(device));
  cudaDeviceProp prop;
  B2_CUDA(cudaGetDeviceProperties(&prop, device));
  if (prop.major != 9 || prop.minor != 0) {
    set_error("device %d is sm_%d%d; libb2gram is built for sm_90a (H100) only", device, prop.major, prop.minor);
    return B2_E_UNSUPPORTED;
  }
  b2_ctx* ctx = new (std::nothrow) b2_ctx();
  if (ctx == nullptr) { set_error("out of host memory"); return B2_E_STATE; }
  ctx->device = device;
  ctx->sm_count = prop.multiProcessorCount;
  ctx->hbm_bytes = prop.totalGlobalMem;
  snprintf(ctx->name, sizeof(ctx->name), "%s", prop.name);
  if (int r = ctx_allocate(ctx)) {   // streams, events, scratch: release whatever was created before the failure
    b2_ctx_destroy(ctx);
    return r;
  }
  *out = ctx;
  return B2_OK;
}

int b2_ctx_destroy(b2_ctx* ctx) {
  if (ctx == nullptr) return B2_OK;
  cudaSetDevice(ctx->device);
  cudaDeviceSynchronize();
  if (ctx->comm != nullptr) b2_comm_destroy(ctx);
  b2_comm_p2p_detach(ctx);
  if (ctx->xchg != nullptr) cudaFree(ctx->xchg);
  void* bufs[] = {ctx->S, ctx->tc_part, ctx->tc_red, ctx->shift, ctx->simt_part, ctx->score_part,
                  ctx->coef_dev, ctx->solve_out, ctx->stage_x[0], ctx->stage_x[1], ctx->stage_y[0], ctx->stage_y[1],
                  ctx->stage_m[0], ctx->stage_m[1], ctx->row_out[0], ctx->row_out[1], ctx->tc_sync, ctx->synth_count,
                  ctx->grad_part, ctx->refine, ctx->loo, ctx->loo_part, ctx->enet, ctx->folds, ctx->fold_range, ctx->glm, ctx->glm_part,
                  ctx->cls, ctx->loo_cls, ctx->mn_op, ctx->mn_sum, ctx->mn_part, ctx->disc, ctx->disc_part,
                  ctx->qda, ctx->qda_hd, ctx->qda_scratch, ctx->qda_part};
  for (void* p : bufs) if (p != nullptr) cudaFree(p);
  if (ctx->solve_host != nullptr) cudaFreeHost(ctx->solve_host);
  if (ctx->xchg_status_host != nullptr) cudaFreeHost(ctx->xchg_status_host);
  if (ctx->coef_host != nullptr) cudaFreeHost(ctx->coef_host);
  for (int b = 0; b < 2; ++b) {
    if (ctx->bounce[b] != nullptr) cudaFreeHost(ctx->bounce[b]);
    if (ctx->ev_bounce[b] != nullptr) cudaEventDestroy(ctx->ev_bounce[b]);
  }
  for (int b = 0; b < 2; ++b) if (ctx->ev_coef[b]) cudaEventDestroy(ctx->ev_coef[b]);
  for (int b = 0; b < 2; ++b) {
    if (ctx->ev_copied[b]) cudaEventDestroy(ctx->ev_copied[b]);
    if (ctx->ev_consumed[b]) cudaEventDestroy(ctx->ev_consumed[b]);
  }
  for (int i = 0; i < kKernelEventPairs; ++i)
    for (int e = 0; e < 2; ++e)
      if (ctx->ev_k[i][e] != nullptr) cudaEventDestroy(ctx->ev_k[i][e]);
  if (ctx->ev_t0 != nullptr) cudaEventDestroy(ctx->ev_t0);
  if (ctx->ev_t1 != nullptr) cudaEventDestroy(ctx->ev_t1);
  if (ctx->stream != nullptr) cudaStreamDestroy(ctx->stream);
  if (ctx->copy_stream != nullptr) cudaStreamDestroy(ctx->copy_stream);
  cudaGetLastError();   // a half-built context may have left a sticky-free error code behind
  delete ctx;
  return B2_OK;
}

int b2_ctx_sync(b2_ctx* ctx) {
  if (int r = use_device(ctx)) return r;
  B2_CUDA(cudaStreamSynchronize(ctx->copy_stream));
  B2_CUDA(cudaStreamSynchronize(ctx->stream));
  return B2_OK;
}

int b2_ctx_info(b2_ctx* ctx, char* name, int name_cap, int* sm_count, size_t* hbm_bytes) {
  if (ctx == nullptr) { set_error("null context"); return B2_E_ARG; }
  if (name != nullptr && name_cap > 0) snprintf(name, (size_t)name_cap, "%s", ctx->name);
  if (sm_count != nullptr) *sm_count = ctx->sm_count;
  if (hbm_bytes != nullptr) *hbm_bytes = ctx->hbm_bytes;
  return B2_OK;
}

int b2_ctx_set_kernel(b2_ctx* ctx, int kernel) {
  if (ctx == nullptr || kernel < B2_KERNEL_AUTO || kernel > B2_KERNEL_NARROW) { set_error("bad kernel id"); return B2_E_ARG; }
  ctx->kernel_mode = kernel;
  return B2_OK;
}

int b2_ctx_set_drain_rows(b2_ctx* ctx, int rows) {
  if (ctx == nullptr || rows < kTcRows || rows % kTcRows != 0) { set_error("drain_rows must be a positive multiple of %d", kTcRows); return B2_E_ARG; }
  ctx->drain_rows = rows;
  return B2_OK;
}

int b2_ctx_set_sm_limit(b2_ctx* ctx, int n_sms) {
  if (ctx == nullptr || n_sms < 0) { set_error("n_sms must be >= 0 (0 = all SMs)"); return B2_E_ARG; }
  ctx->sm_limit = n_sms;
  ctx->sm_limit_auto = false;
  return B2_OK;
}

int b2_ctx_set_precision(b2_ctx* ctx, int precision) {
  if (ctx == nullptr || (precision != B2_PRECISION_SPLIT && precision != B2_PRECISION_BF16)) {
    set_error("precision must be B2_PRECISION_SPLIT or B2_PRECISION_BF16");
    return B2_E_ARG;
  }
  ctx->precision = precision;
  return B2_OK;
}

// ---- buffers ------------------------------------------------------------------------------------
int b2_dev_alloc(b2_ctx* ctx, size_t bytes, void** out) {
  if (int r = use_device(ctx)) return r;
  if (out == nullptr) { set_error("out is null"); return B2_E_ARG; }
  B2_CUDA(cudaMalloc(out, bytes ? bytes : 1));
  return B2_OK;
}
int b2_dev_free(b2_ctx* ctx, void* p) {
  if (int r = use_device(ctx)) return r;
  B2_CUDA(cudaFree(p));
  return B2_OK;
}
int b2_host_alloc(b2_ctx* ctx, size_t bytes, void** out) {
  if (int r = use_device(ctx)) return r;
  if (out == nullptr) { set_error("out is null"); return B2_E_ARG; }
  B2_CUDA(cudaHostAlloc(out, bytes ? bytes : 1, cudaHostAllocDefault));
  return B2_OK;
}
int b2_host_free(b2_ctx* ctx, void* p) {
  if (int r = use_device(ctx)) return r;
  B2_CUDA(cudaFreeHost(p));
  return B2_OK;
}
int b2_copy_h2d(b2_ctx* ctx, void* dst, const void* src, size_t bytes) {
  if (int r = use_device(ctx)) return r;
  B2_CUDA(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyHostToDevice, ctx->stream));
  B2_CUDA(cudaStreamSynchronize(ctx->stream));
  return B2_OK;
}
// ---- DataFrame columns -> row-major fp32 rows in HBM --------------------------------------------------------------------
// pandas keeps every column of `data` as its own strided array; `data[cols].to_numpy(dtype=float32)` + ascontiguousarray
// is two single-threaded passes (a transposing copy and a conversion) and then a pageable H2D copy -- 90 % of train_model's
// time once the fit takes a millisecond.  Here the host threads of the bounce ring gather 16 columns at a time into the
// pinned bounce block (full 64-byte lines written, every column read as its own sequential stream), converting on the fly,
// while the previous block is on the wire.
// the gather + conversion alone, host to host (no device needed): rows [0, n_rows) of d strided columns -> out[n_rows][d]
static int pack_columns_threads(float* dst, const void* const* cols, const int64_t* strides, int dtype, int64_t r0, int64_t rows,
                                int d) {
  const int nt = copy_threads();
  auto work = [=](int t) {
    const int64_t lo = rows * t / nt / 64 * 64, hi = (t == nt - 1) ? rows : rows * (t + 1) / nt / 64 * 64;
    if (hi <= lo) return;
    if (dtype == B2_F64) pack_rows<double>(dst + (size_t)lo * d, cols, strides, r0 + lo, hi - lo, d);
    else pack_rows<float>(dst + (size_t)lo * d, cols, strides, r0 + lo, hi - lo, d);
  };
  if (rows < 4096 || nt == 1) {
    if (dtype == B2_F64) pack_rows<double>(dst, cols, strides, r0, rows, d); else pack_rows<float>(dst, cols, strides, r0, rows, d);
    return B2_OK;
  }
  std::vector<std::thread> pool;
  pool.reserve(nt - 1);
  for (int t = 1; t < nt; ++t) pool.emplace_back(work, t);
  work(0);
  for (auto& th : pool) th.join();
  return B2_OK;
}

int b2_pack_columns(const void* const* cols, const int64_t* strides, int dtype, int64_t n_rows, int d, float* out) {
  if (cols == nullptr || strides == nullptr || out == nullptr || n_rows < 0 || d < 1 || d > kMaxD ||
      (dtype != B2_F32 && dtype != B2_F64)) {
    set_error("b2_pack_columns: bad arguments (1 <= d <= %d, dtype B2_F32 or B2_F64)", kMaxD);
    return B2_E_ARG;
  }
  for (int j = 0; j < d; ++j)
    if (cols[j] == nullptr) { set_error("b2_pack_columns: column %d is null", j); return B2_E_ARG; }
  return pack_columns_threads(out, cols, strides, dtype, 0, n_rows, d);
}

int b2_upload_columns(b2_ctx* ctx, const void* const* cols, const int64_t* strides, int dtype, int64_t n_rows, int d,
                      float* X_dev) {
  if (int r = use_device(ctx)) return r;
  if (cols == nullptr || strides == nullptr || X_dev == nullptr || n_rows < 0 || d < 1 || d > kMaxD ||
      (dtype != B2_F32 && dtype != B2_F64)) {
    set_error("b2_upload_columns: bad arguments (1 <= d <= %d, dtype B2_F32 or B2_F64)", kMaxD);
    return B2_E_ARG;
  }
  for (int j = 0; j < d; ++j)
    if (cols[j] == nullptr) { set_error("b2_upload_columns: column %d is null", j); return B2_E_ARG; }
  if (int r = ensure_staging(ctx)) return r;
  if (int r = ensure_bounce(ctx)) return r;
  int buf = 0;
  for (int64_t r0 = 0; r0 < n_rows; r0 += ctx->stage_rows, buf ^= 1) {
    const int64_t rows = n_rows - r0 < ctx->stage_rows ? n_rows - r0 : ctx->stage_rows;
    B2_CUDA(cudaEventSynchronize(ctx->ev_bounce[buf]));               // the H2D that last read this bounce block is done
    float* dst = static_cast<float*>(ctx->bounce[buf]);
    pack_columns_threads(dst, cols, strides, dtype, r0, rows, d);
    B2_CUDA(cudaMemcpyAsync(X_dev + (size_t)r0 * d, dst, (size_t)rows * d * sizeof(float), cudaMemcpyHostToDevice, ctx->copy_stream));
    B2_CUDA(cudaEventRecord(ctx->ev_bounce[buf], ctx->copy_stream));
  }
  B2_CUDA(cudaStreamSynchronize(ctx->copy_stream));
  return B2_OK;
}

int b2_copy_d2h(b2_ctx* ctx, void* dst, const void* src, size_t bytes) {
  if (int r = use_device(ctx)) return r;
  B2_CUDA(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToHost, ctx->stream));
  B2_CUDA(cudaStreamSynchronize(ctx->stream));
  return B2_OK;
}
int b2_copy_d2d(b2_ctx* ctx, void* dst, const void* src, size_t bytes) {
  if (int r = use_device(ctx)) return r;
  B2_CUDA(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToDevice, ctx->stream));   // asynchronous: ordered on the stream
  return B2_OK;
}
int b2_dev_memset(b2_ctx* ctx, void* dst, int value, size_t bytes) {
  if (int r = use_device(ctx)) return r;
  B2_CUDA(cudaMemsetAsync(dst, value, bytes, ctx->stream));
  return B2_OK;
}

// ---- Gram -----------------------------------------------------------------------------------------
int b2_gram_reset(b2_ctx* ctx, int d) {
  if (int r = use_device(ctx)) return r;
  if (d < 1 || d > kMaxD) { set_error("d=%d out of range [1,%d]", d, kMaxD); return B2_E_ARG; }
  ctx->d = d;
  ctx->s_zero_pending = true;   // the first kernel that writes S overwrites it: no memset launch
  return B2_OK;
}

int b2_gram_accumulate(b2_ctx* ctx, const void* X, int x_dtype, const float* y, int64_t n_rows, int d, int64_t ldx,
                       int mem_kind, const uint8_t* row_mask, int mask_keep) {
  if (int r = use_device(ctx)) return r;
  if (int r = check_shape(x_dtype, n_rows, d, ldx, mem_kind)) return r;
  if (ctx->d == 0) { set_error("b2_gram_reset has not been called"); return B2_E_STATE; }
  if (d != ctx->d) { set_error("d=%d differs from the statistic's d=%d", d, ctx->d); return B2_E_ARG; }
  if (n_rows > 0 && (X == nullptr || y == nullptr)) { set_error("X / y is null"); return B2_E_ARG; }
  return gram_rows(ctx, X, x_dtype, y, n_rows, d, ldx, mem_kind, row_mask, mask_keep);
}

// The peer-memory exchange reports a peer that did not deliver within the timeout through a status word in the
// exchange buffer; it is read together with the next result the host fetches, so a late or dead rank turns into
// B2_E_COMM instead of a fit on a partial statistic.  Call after the stream has been synchronised.
static int queue_exchange_status_read(b2_ctx* ctx) {
  if (!ctx->xchg_pending || ctx->xchg == nullptr) return B2_OK;
  B2_CUDA(cudaMemcpyAsync(ctx->xchg_status_host, xchg_flags(ctx->xchg) + kXchgStatusWord, sizeof(unsigned int),
                          cudaMemcpyDeviceToHost, ctx->stream));
  return B2_OK;
}
static int check_exchange_status(b2_ctx* ctx) {
  if (!ctx->xchg_pending || ctx->xchg == nullptr) return B2_OK;
  ctx->xchg_pending = false;
  const unsigned int st = ctx->xchg_status_host[0];
  if (st != 0u) {
    ctx->xchg_status_host[0] = 0u;
    cudaMemsetAsync(xchg_flags(ctx->xchg) + kXchgStatusWord, 0, sizeof(unsigned int), ctx->stream);
    set_error("peer-memory exchange %u timed out after %.1f s: a rank did not deliver its partial statistic "
              "(S on this rank is incomplete)", st, (double)ctx->xchg_timeout_ns * 1e-9);
    return B2_E_COMM;
  }
  return B2_OK;
}

int b2_gram_allreduce(b2_ctx* ctx) {
  if (int r = use_device(ctx)) return r;
  if (ctx->d == 0) { set_error("b2_gram_reset has not been called"); return B2_E_STATE; }
  if (int r = ensure_s_cleared(ctx)) return r;
  if (ctx->n_ranks > 1 && ctx->p2p_ready) return launch_p2p_allreduce(ctx);   // peer-memory one-shot exchange
  if (ctx->comm == nullptr) return B2_OK;
  NcclApi* api = nccl();
  if (api == nullptr) { set_error("libnccl.so.2 could not be loaded"); return B2_E_COMM; }
  const size_t count = (size_t)(ctx->d + 2) * (ctx->d + 2);
  B2_NCCL(api, api->AllReduce(ctx->S, ctx->S, count, kNcclFloat64, kNcclSum, ctx->comm, ctx->stream));
  return B2_OK;
}

int b2_gram_export(b2_ctx* ctx, double* S_out, int64_t* n_rows_out) {
  if (int r = use_device(ctx)) return r;
  if (ctx->d == 0) { set_error("b2_gram_reset has not been called"); return B2_E_STATE; }
  const int dp = ctx->d + 2;
  if (S_out == nullptr) { set_error("S_out is null"); return B2_E_ARG; }
  if (int r = ensure_s_cleared(ctx)) return r;
  B2_CUDA(cudaMemcpyAsync(S_out, ctx->S, sizeof(double) * dp * dp, cudaMemcpyDeviceToHost, ctx->stream));
  if (int r = queue_exchange_status_read(ctx)) return r;
  B2_CUDA(cudaStreamSynchronize(ctx->stream));
  if (int r = check_exchange_status(ctx)) return r;
  if (n_rows_out != nullptr) *n_rows_out = (int64_t)(S_out[ctx->d * dp + ctx->d] + 0.5);
  return B2_OK;
}

int b2_gram_import(b2_ctx* ctx, const double* S_in, int d) {
  if (int r = use_device(ctx)) return r;
  if (d < 1 || d > kMaxD || S_in == nullptr) { set_error("bad arguments to b2_gram_import"); return B2_E_ARG; }
  ctx->d = d;
  ctx->s_zero_pending = false;
  B2_CUDA(cudaMemsetAsync(ctx->S, 0, sizeof(double) * kMaxS * kMaxS, ctx->stream));
  B2_CUDA(cudaMemcpyAsync(ctx->S, S_in, sizeof(double) * (d + 2) * (d + 2), cudaMemcpyHostToDevice, ctx->stream));
  B2_CUDA(cudaStreamSynchronize(ctx->stream));
  return B2_OK;
}

// ---- solve ------------------------------------------------------------------------------------------
// from_pinned: the Cholesky kernel has written its result into ctx->solve_host itself (no copy node to wait for)
static int fetch_solution(b2_ctx* ctx, bool from_pinned, double* coef, double* intercept, double* singular, int* rank,
                          double* info) {
  double* host = ctx->solve_host;
  if (!from_pinned)
    B2_CUDA(cudaMemcpyAsync(host, ctx->solve_out, sizeof(double) * (2 * kMaxD + 8), cudaMemcpyDeviceToHost, ctx->stream));
  if (int r = queue_exchange_status_read(ctx)) return r;
  B2_CUDA(cudaStreamSynchronize(ctx->stream));
  if (int r = check_exchange_status(ctx)) return r;
  if (coef != nullptr) memcpy(coef, host, sizeof(double) * ctx->d);
  if (intercept != nullptr) *intercept = host[kMaxD];
  *info = host[kMaxD + 1];
  if (rank != nullptr) *rank = (int)host[kMaxD + 2];
  if (singular != nullptr) memcpy(singular, host + kMaxD + 3, sizeof(double) * ctx->d);
  return B2_OK;
}

static int finish_cholesky(b2_ctx* ctx, double* coef, double* intercept) {
  double info = 0.0;
#ifdef B2_DEV_KNOBS
  double phase[kMaxD];
  if (int r = fetch_solution(ctx, true, coef, intercept, getenv("B2_SOLVE_TIMING") ? phase : nullptr, nullptr, &info)) return r;
  if (getenv("B2_SOLVE_TIMING"))
    fprintf(stderr, "[b2_solve] cycles: build %.0f diag %.0f panel %.0f update %.0f backward %.0f\n", phase[0], phase[1],
            phase[2], phase[3], phase[4]);
#else
  if (int r = fetch_solution(ctx, true, coef, intercept, nullptr, nullptr, &info)) return r;
#endif
  if (info < 0.0) {
    ctx->xchg_pending = false;
    set_error("peer-memory exchange timed out after %.1f s inside the solve: a rank did not deliver its partial "
              "statistic", (double)ctx->xchg_timeout_ns * 1e-9);
    cudaMemsetAsync(xchg_flags(ctx->xchg) + kXchgStatusWord, 0, sizeof(unsigned int), ctx->stream);
    return B2_E_COMM;
  }
  if (info != 0.0) {
    set_error("pivot %d of the LDL^T factorisation is not positive: the centred Gram matrix is rank deficient "
              "(use alpha > 0 or b2_solve_spectral)", (int)info);
    return B2_E_SINGULAR;
  }
  return B2_OK;
}

int b2_solve(b2_ctx* ctx, double alpha, int fit_intercept, double* coef, double* intercept) {
  if (int r = use_device(ctx)) return r;
  if (ctx->d == 0) { set_error("b2_gram_reset has not been called"); return B2_E_STATE; }
  if (!(alpha >= 0.0)) { set_error("alpha must be >= 0"); return B2_E_ARG; }
  if (int r = ensure_s_cleared(ctx)) return r;
  if (int r = launch_solve_cholesky(ctx, alpha, fit_intercept)) return r;
  return finish_cholesky(ctx, coef, intercept);
}

int b2_solve_spectral(b2_ctx* ctx, double cond, int fit_intercept, double* coef, double* intercept, double* singular,
                      int* rank) {
  if (int r = use_device(ctx)) return r;
  if (ctx->d == 0) { set_error("b2_gram_reset has not been called"); return B2_E_STATE; }
  if (int r = ensure_s_cleared(ctx)) return r;
  if (int r = launch_solve_spectral(ctx, cond, fit_intercept)) return r;
  double info = 0.0;
  return fetch_solution(ctx, false, coef, intercept, singular, rank, &info);
}

int b2_solve_eigvals(b2_ctx* ctx, double cond, int fit_intercept, double* singular, int* rank, int64_t* n_rows_out) {
  if (int r = use_device(ctx)) return r;
  if (ctx->d == 0) { set_error("b2_gram_reset has not been called"); return B2_E_STATE; }
  if (int r = ensure_s_cleared(ctx)) return r;
  if (int r = launch_solve_eigvals(ctx, cond, fit_intercept)) return r;
  double info = 0.0;
  if (int r = fetch_solution(ctx, false, nullptr, nullptr, singular, rank, &info)) return r;
  if (n_rows_out != nullptr) *n_rows_out = (int64_t)(ctx->solve_host[kMaxD + 3 + kMaxD] + 0.5);
#ifdef B2_DEV_KNOBS
  if (getenv("B2_SOLVE_TIMING")) {
    const double* t = ctx->solve_host + kMaxD + 3 + kMaxD + 1;
    fprintf(stderr, "[b2_solve_eigvals] cycles: build %.0f tridiagonalise %.0f scale %.0f multisection %.0f\n", t[0], t[1], t[2], t[3]);
  }
#endif
  return B2_OK;
}

// ---- the whole fit in one call ----------------------------------------------------------------------------
// reset + accumulate + all-reduce + solve.  With an attached peer exchange and device rows whose final Gram launch is
// tensor-core, the exchange rides on the kernels: the finalize kernel stores S straight into the peers' exchange slots,
// and the solve kernel waits for them and sums them before it factors.  Otherwise the stand-alone exchange of
// b2_gram_allreduce runs before the solve.  The solve kernel writes the coefficients into pinned host memory.
int b2_fit(b2_ctx* ctx, const void* X, int x_dtype, const float* y, int64_t n_rows, int d, int64_t ldx, int mem_kind,
           const uint8_t* row_mask, int mask_keep, double alpha, int fit_intercept, double* coef, double* intercept) {
  if (int r = use_device(ctx)) return r;
  if (int r = check_shape(x_dtype, n_rows, d, ldx, mem_kind)) return r;
  if (!(alpha >= 0.0)) { set_error("alpha must be >= 0"); return B2_E_ARG; }
  if (n_rows > 0 && (X == nullptr || y == nullptr)) { set_error("X / y is null"); return B2_E_ARG; }
  if (int r = b2_gram_reset(ctx, d)) return r;
  unsigned int gather_epoch = 0;
  if (mem_kind == B2_MEM_DEVICE) {
    bool tc_last = false;
    if (int r = gram_dispatch(ctx, X, x_dtype, y, n_rows, d, ldx, row_mask, mask_keep, &tc_last, &gather_epoch))
      return r;
    if (tc_last) ctx->fused_fits += 1;
  } else if (int r = gram_rows(ctx, X, x_dtype, y, n_rows, d, ldx, mem_kind, row_mask, mask_keep)) {
    return r;
  }
  if (gather_epoch == 0) {
    if (int r = b2_gram_allreduce(ctx)) return r;
  }
  if (int r = launch_solve_cholesky(ctx, alpha, fit_intercept, gather_epoch)) return r;
  return finish_cholesky(ctx, coef, intercept);
}

// One residual pass over the rows for the model in ctx->refine: the gradient kernels (+ their ordered reduce) write
// g_j, g_1 and sum e^2 to ctx->refine + kRfGrad; host rows re-stream through the staging ring.
static int grad_pass(b2_ctx* ctx, const void* X, int x_dtype, const float* y, int64_t n_rows, int d, int64_t ldx,
                     int mem_kind, const uint8_t* row_mask, int mask_keep) {
  return row_pass(ctx, X, x_dtype, y, n_rows, d, ldx, mem_kind, row_mask, [&](const RowSpan& s, void*, void*, void*) {
    return launch_grad(ctx, s.X, x_dtype, s.rows, d, s.ldx, s.y, s.mask, mask_keep, s.first);
  });
}

// The model b0' + (x - m).beta of the residual passes into ctx->refine, with beta = coef and m the column means of the
// resident S (0 without an intercept), also as the state before the last correction (step +inf).  intercept null: b0'
// is S's mean label (0 without an intercept), the state of the fit of S; otherwise b0' = *intercept + m.beta, the model
// *intercept + x.beta.  The upload is from pageable memory, so it has read the state when this returns.
static int load_refine_state(b2_ctx* ctx, int d, const double* coef, int fit_intercept, const double* intercept) {
  if (int r = ensure_s_cleared(ctx)) return r;
  const int dp = d + 2;
  std::vector<double> S((size_t)dp * dp), st(kRfDoubles, 0.0);
  B2_CUDA(cudaMemcpyAsync(S.data(), ctx->S, sizeof(double) * dp * dp, cudaMemcpyDeviceToHost, ctx->stream));
  B2_CUDA(cudaStreamSynchronize(ctx->stream));
  const double n = S[(size_t)d * dp + d];
  const double inv_n = n > 0.0 ? 1.0 / n : 0.0;
  double b0 = intercept != nullptr ? *intercept : (fit_intercept ? S[(size_t)d * dp + d + 1] * inv_n : 0.0);
  for (int j = 0; j < d; ++j) {
    st[kRfBeta + j] = st[kRfPrevBeta + j] = coef[j];
    st[kRfMean + j] = fit_intercept ? S[(size_t)j * dp + d] * inv_n : 0.0;
    if (intercept != nullptr) b0 += st[kRfMean + j] * coef[j];
  }
  st[kRfB0] = st[kRfPrevB0] = b0;
  st[kRfStep] = INFINITY;
  B2_CUDA(cudaMemcpyAsync(ctx->refine, st.data(), sizeof(double) * kRfDoubles, cudaMemcpyHostToDevice, ctx->stream));
  return B2_OK;
}

// ---- the refined fit: b2_fit, then residual passes over the same rows (DESIGN.md section 2) ------------------------
// Per pass: the gradient kernels (+ their ordered reduce) over the rows -- host rows re-stream through the staging ring --
// then the Cholesky kernel in refinement mode, which refactors A + alpha I from S, solves for the correction and moves
// the state; one host synchronisation reads the step and the guard.
int b2_fit_refined(b2_ctx* ctx, const void* X, int x_dtype, const float* y, int64_t n_rows, int d, int64_t ldx,
                   int mem_kind, const uint8_t* row_mask, int mask_keep, double alpha, int fit_intercept, int max_passes,
                   double tol, double* coef, double* intercept, int* passes_out, double* step_out) {
  if (int r = use_device(ctx)) return r;
  if (int r = check_shape(x_dtype, n_rows, d, ldx, mem_kind)) return r;
  if (max_passes < 0 || max_passes > 16) { set_error("max_passes=%d out of range [0,16]", max_passes); return B2_E_ARG; }
  if (!(tol >= 0.0)) { set_error("tol must be >= 0"); return B2_E_ARG; }
  if (coef == nullptr || intercept == nullptr) { set_error("coef / intercept is null"); return B2_E_ARG; }
  if (ctx->n_ranks > 1) {
    set_error("b2_fit_refined runs on one rank only (the residual gradient is not exchanged between ranks)");
    return B2_E_UNSUPPORTED;
  }
  if (passes_out != nullptr) *passes_out = 0;
  if (step_out != nullptr) *step_out = 0.0;
  if (int r = b2_fit(ctx, X, x_dtype, y, n_rows, d, ldx, mem_kind, row_mask, mask_keep, alpha, fit_intercept, coef,
                     intercept))
    return r;
  if (max_passes == 0) return B2_OK;
  // the state: beta from the fit; m and b0' from S as the solve forms them
  if (int r = load_refine_state(ctx, d, coef, fit_intercept, nullptr)) return r;
  B2_CUDA(cudaStreamSynchronize(ctx->stream));
  const double* h = ctx->solve_host;
  int kept = 0;
  for (int pass = 0; pass < max_passes; ++pass) {
    if (int r = grad_pass(ctx, X, x_dtype, y, n_rows, d, ldx, mem_kind, row_mask, mask_keep)) return r;
    if (int r = launch_solve_refine(ctx, alpha, fit_intercept)) return r;
    B2_CUDA(cudaStreamSynchronize(ctx->stream));
    if (h[kMaxD + 1] != 0.0) {
      set_error("pivot %d of the LDL^T factorisation is not positive in a refinement pass", (int)h[kMaxD + 1]);
      return B2_E_SINGULAR;
    }
    if (step_out != nullptr) *step_out = h[kOutRefineStep];
    if (h[kOutRefineGuard] != 0.0) {         // the state went back to before the last kept correction
      kept = kept > 0 ? kept - 1 : 0;
      break;
    }
    ++kept;
    if (h[kOutRefineStep] <= tol) break;
  }
  memcpy(coef, h, sizeof(double) * d);
  *intercept = h[kMaxD];
  if (passes_out != nullptr) *passes_out = kept;
  return B2_OK;
}

// the Jacobi kernel's convergence flag (ctx->loo + kLooMisc + 3) as a return code
static int eigh_converged(double flag) {
  if (flag != 0.0) return B2_OK;
  set_error("the Jacobi eigendecomposition did not converge within its sweep limit");
  return B2_E_SINGULAR;
}

// ---- eigendecomposition and RidgeCV's leave-one-out error (DESIGN.md section 6) ---------------------------------
int b2_solve_eigh(b2_ctx* ctx, int fit_intercept, double* eigvals, double* eigvecs) {
  if (int r = use_device(ctx)) return r;
  if (ctx->d == 0) { set_error("b2_gram_reset has not been called"); return B2_E_STATE; }
  if (int r = ensure_s_cleared(ctx)) return r;
  if (int r = launch_solve_eigh(ctx, fit_intercept)) return r;
  const int d = ctx->d;
  double converged = 0.0;
  B2_CUDA(cudaMemcpyAsync(&converged, ctx->loo + kLooMisc + 3, sizeof(double), cudaMemcpyDeviceToHost, ctx->stream));
  if (eigvals != nullptr)
    B2_CUDA(cudaMemcpyAsync(eigvals, ctx->loo + kLooLam, sizeof(double) * d, cudaMemcpyDeviceToHost, ctx->stream));
  if (eigvecs != nullptr)
    B2_CUDA(cudaMemcpy2DAsync(eigvecs, sizeof(double) * d, ctx->loo + kLooQ, sizeof(double) * kMaxD, sizeof(double) * d, d,
                              cudaMemcpyDeviceToHost, ctx->stream));
  B2_CUDA(cudaStreamSynchronize(ctx->stream));
  return eigh_converged(converged);
}

// ---- ElasticNet / Lasso: the coordinate-descent path of the resident S (DESIGN.md section 7) -------------------------
// The argument checks of b2_solve_enet_path and b2_solve_enet_cv (n_l1 l1_ratios, host arrays).
static int check_enet_args(const double* l1_ratios, int n_l1, const double* alphas, int n_alphas, double eps,
                           int max_iter, double tol) {
  for (int l = 0; l < n_l1; ++l) {
    const double l1_ratio = l1_ratios[l];
    if (!(l1_ratio >= 0.0 && l1_ratio <= 1.0)) { set_error("l1_ratio=%g must be in [0, 1]", l1_ratio); return B2_E_ARG; }
    if (alphas == nullptr && l1_ratio == 0.0) {
      set_error("Automatic alpha grid generation is not supported for l1_ratio=0. Please supply a grid by providing "
                "your estimator with the appropriate `alphas=` argument.");
      return B2_E_ARG;
    }
  }
  if (n_alphas < 1) { set_error("n_alphas=%d must be >= 1", n_alphas); return B2_E_ARG; }
  if (alphas == nullptr && !(eps > 0.0 && isfinite(eps))) { set_error("eps=%g must be > 0 and finite", eps); return B2_E_ARG; }
  if (alphas != nullptr)
    for (int a = 0; a < n_alphas; ++a)
      if (!(isfinite(alphas[a]) && alphas[a] >= 0.0)) {
        set_error("alphas[%d] == %g, must be >= 0.0 and finite", a, alphas[a]);
        return B2_E_ARG;
      }
  if (max_iter < 1) { set_error("max_iter=%d must be >= 1", max_iter); return B2_E_ARG; }
  if (!(tol >= 0.0)) { set_error("tol must be >= 0"); return B2_E_ARG; }
  return B2_OK;
}

// ctx->enet grown to `need` doubles (its contents are not kept)
static int ensure_enet_block(b2_ctx* ctx, size_t need) {
  if (ctx->enet_doubles >= need) return B2_OK;
  if (ctx->enet != nullptr) cudaFree(ctx->enet);
  ctx->enet = nullptr;
  ctx->enet_doubles = 0;
  if (cudaMalloc(reinterpret_cast<void**>(&ctx->enet), sizeof(double) * need) != cudaSuccess) {
    cudaGetLastError();
    set_error("out of device memory for the elastic-net paths (%zu doubles)", need);
    return B2_E_CUDA;
  }
  ctx->enet_doubles = need;
  return B2_OK;
}

// Host checks, the inputs into ctx->enet, one launch, the outputs back.  ctx->enet holds
// [alphas A | coef_init kMaxD | coefs A x d | intercepts A | gaps A | iters A | tol_out 1] and grows to the largest call.
int b2_solve_enet_path(b2_ctx* ctx, int fit_intercept, double l1_ratio, const double* alphas, int n_alphas, double eps,
                       int max_iter, double tol, int positive, const double* coef_init, double* alphas_out,
                       double* coefs_out, double* intercepts_out, double* gaps_out, int* n_iter_out, double* tol_out) {
  if (int r = use_device(ctx)) return r;
  if (ctx->d == 0) { set_error("b2_gram_reset has not been called"); return B2_E_STATE; }
  if (int r = check_enet_args(&l1_ratio, 1, alphas, n_alphas, eps, max_iter, tol)) return r;
  if (alphas_out == nullptr || coefs_out == nullptr || intercepts_out == nullptr || gaps_out == nullptr ||
      n_iter_out == nullptr) {
    set_error("alphas_out / coefs_out / intercepts_out / gaps_out / n_iter_out is null");
    return B2_E_ARG;
  }
  if (int r = ensure_s_cleared(ctx)) return r;
  const int d = ctx->d;
  double n = 0.0;
  B2_CUDA(cudaMemcpyAsync(&n, ctx->S + (size_t)d * (d + 2) + d, sizeof(double), cudaMemcpyDeviceToHost, ctx->stream));
  B2_CUDA(cudaStreamSynchronize(ctx->stream));
  if (!(n > 0.0)) { set_error("no row kept: the statistic holds no rows"); return B2_E_ARG; }
  const size_t A = (size_t)n_alphas;
  if (int r = ensure_enet_block(ctx, A + kMaxD + A * d + 3 * A + 1)) return r;
  EnetArgs args;
  args.l1_ratio = l1_ratio;
  args.eps = eps;
  args.tol = tol;
  args.n_alphas = n_alphas;
  args.grid = alphas == nullptr ? 1 : 0;
  args.max_iter = max_iter;
  args.positive = positive ? 1 : 0;
  args.fit_intercept = fit_intercept ? 1 : 0;
  args.alphas = ctx->enet;
  args.coef_init = coef_init != nullptr ? ctx->enet + A : nullptr;
  args.coefs = ctx->enet + A + kMaxD;
  args.intercepts = args.coefs + A * d;
  args.gaps = args.intercepts + A;
  args.iters = args.gaps + A;
  args.tol_out = args.iters + A;
  if (alphas != nullptr)
    B2_CUDA(cudaMemcpyAsync(args.alphas, alphas, sizeof(double) * A, cudaMemcpyHostToDevice, ctx->stream));
  if (coef_init != nullptr)
    B2_CUDA(cudaMemcpyAsync(ctx->enet + A, coef_init, sizeof(double) * d, cudaMemcpyHostToDevice, ctx->stream));
  if (int r = launch_solve_enet(ctx, args)) return r;
  std::vector<double> iters(A);
  double tol_abs = 0.0;
  B2_CUDA(cudaMemcpyAsync(alphas_out, args.alphas, sizeof(double) * A, cudaMemcpyDeviceToHost, ctx->stream));
  B2_CUDA(cudaMemcpyAsync(coefs_out, args.coefs, sizeof(double) * A * d, cudaMemcpyDeviceToHost, ctx->stream));
  B2_CUDA(cudaMemcpyAsync(intercepts_out, args.intercepts, sizeof(double) * A, cudaMemcpyDeviceToHost, ctx->stream));
  B2_CUDA(cudaMemcpyAsync(gaps_out, args.gaps, sizeof(double) * A, cudaMemcpyDeviceToHost, ctx->stream));
  B2_CUDA(cudaMemcpyAsync(iters.data(), args.iters, sizeof(double) * A, cudaMemcpyDeviceToHost, ctx->stream));
  B2_CUDA(cudaMemcpyAsync(&tol_abs, args.tol_out, sizeof(double), cudaMemcpyDeviceToHost, ctx->stream));
  B2_CUDA(cudaStreamSynchronize(ctx->stream));
  for (size_t a = 0; a < A; ++a) n_iter_out[a] = (int)iters[a];
  if (tol_out != nullptr) *tol_out = tol_abs;
  return B2_OK;
}

// ---- LassoCV / ElasticNetCV: fold statistics and the paths of every (l1_ratio, fold) (DESIGN.md section 8) ------------
// ctx->folds grown to n_folds statistics of (d+2)^2 doubles
static int ensure_folds_block(b2_ctx* ctx, int n_folds, int d) {
  const size_t need = (size_t)n_folds * (d + 2) * (d + 2);
  if (ctx->fold_range == nullptr)
    B2_CUDA(cudaMalloc(reinterpret_cast<void**>(&ctx->fold_range), sizeof(unsigned long long) * 2 * kMaxFolds));
  ctx->n_folds = 0;
  if (ctx->folds_doubles >= need) return B2_OK;
  if (ctx->folds != nullptr) cudaFree(ctx->folds);
  ctx->folds = nullptr;
  ctx->folds_doubles = 0;
  if (cudaMalloc(reinterpret_cast<void**>(&ctx->folds), sizeof(double) * need) != cudaSuccess) {
    cudaGetLastError();
    set_error("out of device memory for %d fold statistics at d=%d", n_folds, d);
    return B2_E_CUDA;
  }
  ctx->folds_doubles = need;
  return B2_OK;
}

int b2_gram_folds(b2_ctx* ctx, const void* X, int x_dtype, const float* y, int64_t n_rows, int d, int64_t ldx,
                  int mem_kind, const uint8_t* fold_of_row, int n_folds, double* fold_S_out) {
  if (int r = use_device(ctx)) return r;
  if (int r = check_shape(x_dtype, n_rows, d, ldx, mem_kind)) return r;
  if (n_folds < 2 || n_folds > kMaxFolds) { set_error("n_folds=%d must be in [2, %d]", n_folds, kMaxFolds); return B2_E_ARG; }
  if (ctx->n_ranks > 1) { set_error("cross-validation folds are computed on one rank only"); return B2_E_UNSUPPORTED; }
  if (n_rows > 0 && (X == nullptr || y == nullptr || fold_of_row == nullptr)) {
    set_error("X / y / fold_of_row is null");
    return B2_E_ARG;
  }
  if (int r = ensure_folds_block(ctx, n_folds, d)) return r;
  // first and last row of every fold
  std::vector<int64_t> first(n_folds, n_rows), last(n_folds, -1);
  if (mem_kind == B2_MEM_DEVICE) {
    std::vector<unsigned long long> rg(2 * n_folds);
    if (int r = launch_fold_ranges(ctx, fold_of_row, n_rows, n_folds, ctx->fold_range)) return r;
    B2_CUDA(cudaMemcpyAsync(rg.data(), ctx->fold_range, sizeof(unsigned long long) * 2 * n_folds, cudaMemcpyDeviceToHost,
                            ctx->stream));
    B2_CUDA(cudaStreamSynchronize(ctx->stream));
    for (int k = 0; k < n_folds; ++k)
      if (rg[2 * k + 1] != 0ull) { first[k] = n_rows - (int64_t)rg[2 * k]; last[k] = (int64_t)rg[2 * k + 1] - 1; }
  } else {
    for (int64_t r = 0; r < n_rows; ++r) {
      const int f = fold_of_row[r];
      if (f < n_folds) {
        if (first[f] > r) first[f] = r;
        last[f] = r;
      }
    }
  }
  for (int k = 0; k < n_folds; ++k)
    if (last[k] < 0) { set_error("fold %d has no rows", k); return B2_E_ARG; }
  // fold k: the Gram dispatch over [first rounded down to 16, last + 1) keeping the rows whose id is k
  const int es = x_dtype == B2_F32 ? 4 : 2;
  const size_t count = (size_t)(d + 2) * (d + 2);
  ctx->d = d;
  for (int k = 0; k < n_folds; ++k) {
    const int64_t r0 = first[k] & ~(int64_t)15, rows = last[k] + 1 - r0;
    const void* Xk = static_cast<const char*>(X) + (size_t)r0 * ldx * es;
    ctx->s_zero_pending = true;
    if (int r = gram_rows(ctx, Xk, x_dtype, y + r0, rows, d, ldx, mem_kind, fold_of_row + r0, k)) return r;
    B2_CUDA(cudaMemcpyAsync(ctx->folds + k * count, ctx->S, sizeof(double) * count, cudaMemcpyDeviceToDevice,
                            ctx->stream));
  }
  if (int r = launch_fold_sum(ctx, ctx->folds, n_folds, d, ctx->S)) return r;
  ctx->s_zero_pending = false;
  ctx->n_folds = n_folds;
  ctx->folds_d = d;
  if (fold_S_out != nullptr) {
    B2_CUDA(cudaMemcpyAsync(fold_S_out, ctx->folds, sizeof(double) * n_folds * count, cudaMemcpyDeviceToHost,
                            ctx->stream));
    B2_CUDA(cudaStreamSynchronize(ctx->stream));
  }
  return B2_OK;
}

// ctx->enet: [alphas n_l1 x A | l1_ratios n_l1 | coefs P x A x d | intercepts P x A | gaps P x A | iters P x A | tol P |
// mse n_l1 x A x K], P = n_l1 K paths
int b2_solve_enet_cv(b2_ctx* ctx, const double* fold_S, int n_folds, int fit_intercept, const double* l1_ratios, int n_l1,
                     const double* alphas, int n_alphas, double eps, int max_iter, double tol, int positive,
                     double* alphas_out, double* mse_out, int* n_iter_out, double* gaps_out, double* coefs_out) {
  if (int r = use_device(ctx)) return r;
  if (ctx->d == 0) { set_error("b2_gram_reset has not been called"); return B2_E_STATE; }
  if (n_folds < 2 || n_folds > kMaxFolds) { set_error("n_folds=%d must be in [2, %d]", n_folds, kMaxFolds); return B2_E_ARG; }
  if (n_l1 < 1 || l1_ratios == nullptr) { set_error("n_l1=%d must be >= 1 with l1_ratios given", n_l1); return B2_E_ARG; }
  if (int r = check_enet_args(l1_ratios, n_l1, alphas, n_alphas, eps, max_iter, tol)) return r;
  if (alphas_out == nullptr || mse_out == nullptr || n_iter_out == nullptr || gaps_out == nullptr) {
    set_error("alphas_out / mse_out / n_iter_out / gaps_out is null");
    return B2_E_ARG;
  }
  const int d = ctx->d;
  const size_t count = (size_t)(d + 2) * (d + 2);
  if (fold_S != nullptr) {
    // designed statistics: the folds uploaded, S their sum in fold order (the additions of fold_sum_kernel)
    for (int k = 0; k < n_folds; ++k)
      if (!(fold_S[k * count + (size_t)d * (d + 2) + d] > 0.0)) { set_error("fold %d has no rows", k); return B2_E_ARG; }
    if (int r = ensure_folds_block(ctx, n_folds, d)) return r;
    std::vector<double> sum(count, 0.0);
    for (int k = 0; k < n_folds; ++k)
      for (size_t i = 0; i < count; ++i) sum[i] += fold_S[k * count + i];
    B2_CUDA(cudaMemcpyAsync(ctx->folds, fold_S, sizeof(double) * n_folds * count, cudaMemcpyHostToDevice, ctx->stream));
    B2_CUDA(cudaMemsetAsync(ctx->S, 0, sizeof(double) * kMaxS * kMaxS, ctx->stream));
    B2_CUDA(cudaMemcpyAsync(ctx->S, sum.data(), sizeof(double) * count, cudaMemcpyHostToDevice, ctx->stream));
    B2_CUDA(cudaStreamSynchronize(ctx->stream));
    ctx->s_zero_pending = false;
    ctx->n_folds = n_folds;
    ctx->folds_d = d;
  } else if (ctx->n_folds != n_folds || ctx->folds_d != d) {
    set_error("no statistics of %d folds at d=%d: call b2_gram_folds first", n_folds, d);
    return B2_E_STATE;
  }
  const size_t A = (size_t)n_alphas, L = (size_t)n_l1, K = (size_t)n_folds, P = L * K;
  if (int r = ensure_enet_block(ctx, L * A + L + P * A * d + 3 * P * A + P + L * A * K)) return r;
  EnetArgs args;
  args.l1_ratio = l1_ratios[0];
  args.eps = eps;
  args.tol = tol;
  args.n_alphas = n_alphas;
  args.grid = alphas == nullptr ? 1 : 0;
  args.max_iter = max_iter;
  args.positive = positive ? 1 : 0;
  args.fit_intercept = fit_intercept ? 1 : 0;
  args.alphas = ctx->enet;
  args.coef_init = nullptr;
  double* l1_dev = ctx->enet + L * A;
  args.coefs = l1_dev + L;
  args.intercepts = args.coefs + P * A * d;
  args.gaps = args.intercepts + P * A;
  args.iters = args.gaps + P * A;
  args.tol_out = args.iters + P * A;
  args.mse = args.tol_out + P;
  args.folds = ctx->folds;
  args.l1_ratios = l1_dev;
  args.n_folds = n_folds;
  args.n_l1 = n_l1;
  if (alphas != nullptr)
    B2_CUDA(cudaMemcpyAsync(args.alphas, alphas, sizeof(double) * A, cudaMemcpyHostToDevice, ctx->stream));
  B2_CUDA(cudaMemcpyAsync(l1_dev, l1_ratios, sizeof(double) * L, cudaMemcpyHostToDevice, ctx->stream));
  if (int r = launch_solve_enet(ctx, args)) return r;
  std::vector<double> iters(P * A);
  if (alphas == nullptr)
    B2_CUDA(cudaMemcpyAsync(alphas_out, args.alphas, sizeof(double) * L * A, cudaMemcpyDeviceToHost, ctx->stream));
  B2_CUDA(cudaMemcpyAsync(mse_out, args.mse, sizeof(double) * L * A * K, cudaMemcpyDeviceToHost, ctx->stream));
  B2_CUDA(cudaMemcpyAsync(gaps_out, args.gaps, sizeof(double) * P * A, cudaMemcpyDeviceToHost, ctx->stream));
  B2_CUDA(cudaMemcpyAsync(iters.data(), args.iters, sizeof(double) * P * A, cudaMemcpyDeviceToHost, ctx->stream));
  if (coefs_out != nullptr)
    B2_CUDA(cudaMemcpyAsync(coefs_out, args.coefs, sizeof(double) * P * A * d, cudaMemcpyDeviceToHost, ctx->stream));
  B2_CUDA(cudaStreamSynchronize(ctx->stream));
  if (alphas != nullptr)
    for (size_t l = 0; l < L; ++l)
      for (size_t a = 0; a < A; ++a) alphas_out[l * A + a] = alphas[a];
  for (size_t i = 0; i < P * A; ++i) n_iter_out[i] = (int)iters[i];
  return B2_OK;
}

// The Gram of b2_fit, the eigendecomposition of its centred Gram, one leave-one-out pass over the same rows (host rows
// re-stream through the staging ring, their e^2 through a device block per row block), then the LDL^T solve of b2_fit
// at the chosen alpha from the same S.
int b2_ridge_loo(b2_ctx* ctx, const void* X, int x_dtype, const float* y, int64_t n_rows, int d, int64_t ldx,
                 int mem_kind, const uint8_t* row_mask, int mask_keep, const double* alphas, int n_alphas,
                 int fit_intercept, double* mse_out, double* cv_out, int* best_out, double* coef, double* intercept) {
  if (int r = use_device(ctx)) return r;
  if (int r = check_shape(x_dtype, n_rows, d, ldx, mem_kind)) return r;
  if (alphas == nullptr || n_alphas < 1 || n_alphas > kMaxAlphas) {
    set_error("n_alphas=%d out of range [1,%d] (or alphas is null)", n_alphas, kMaxAlphas);
    return B2_E_ARG;
  }
  for (int a = 0; a < n_alphas; ++a)
    if (!(isfinite(alphas[a]) && alphas[a] > 0.0)) {
      set_error("alphas[%d] == %g, must be > 0.0 and finite", a, alphas[a]);
      return B2_E_ARG;
    }
  if (mse_out == nullptr || best_out == nullptr || coef == nullptr || intercept == nullptr) {
    set_error("mse_out / best_out / coef / intercept is null");
    return B2_E_ARG;
  }
  if (n_rows > 0 && (X == nullptr || y == nullptr)) { set_error("X / y is null"); return B2_E_ARG; }
  if (ctx->n_ranks > 1) {
    set_error("b2_ridge_loo runs on one rank only (the leave-one-out pass is not exchanged between ranks)");
    return B2_E_UNSUPPORTED;
  }
  if (int r = b2_gram_reset(ctx, d)) return r;
  if (int r = gram_rows(ctx, X, x_dtype, y, n_rows, d, ldx, mem_kind, row_mask, mask_keep)) return r;
  if (int r = ensure_s_cleared(ctx)) return r;
  if (int r = launch_solve_eigh(ctx, fit_intercept)) return r;
  B2_CUDA(cudaMemcpyAsync(ctx->loo + kLooAlpha, alphas, sizeof(double) * n_alphas, cudaMemcpyHostToDevice, ctx->stream));
  double misc[4];
  B2_CUDA(cudaMemcpyAsync(misc, ctx->loo + kLooMisc, sizeof(misc), cudaMemcpyDeviceToHost, ctx->stream));
  B2_CUDA(cudaStreamSynchronize(ctx->stream));
  const double n_kept = misc[1];
  if (!(n_kept > 0.0)) { set_error("no row kept: the leave-one-out error needs at least one row"); return B2_E_ARG; }
  if (int r = eigh_converged(misc[3])) return r;
  if (int r = row_pass(
          ctx, X, x_dtype, y, n_rows, d, ldx, mem_kind, row_mask,
          [&](const RowSpan& s, void* cv, void*, void*) {
            return launch_loo(ctx, s.X, x_dtype, s.rows, d, s.ldx, s.y, s.mask, mask_keep, n_alphas,
                              static_cast<double*>(cv), s.first);
          },
          RowOut{cv_out, sizeof(double) * n_alphas}))
    return r;
  double sums[kMaxAlphas];
  B2_CUDA(cudaMemcpyAsync(sums, ctx->loo + kLooSum, sizeof(double) * n_alphas, cudaMemcpyDeviceToHost, ctx->stream));
  B2_CUDA(cudaStreamSynchronize(ctx->stream));
  int best = 0;
  for (int a = 0; a < n_alphas; ++a) {
    mse_out[a] = sums[a] / n_kept;
    if (mse_out[a] < mse_out[best]) best = a;        // the first of equal minima, as sklearn's argmax of the score
  }
  *best_out = best;
  if (int r = launch_solve_cholesky(ctx, alphas[best], fit_intercept)) return r;
  return finish_cholesky(ctx, coef, intercept);
}

// ---- BayesianRidge / ARDRegression (DESIGN.md section 9) ------------------------------------------------------------
// The anchor pass: the refined fit's gradient kernels at (coef, intercept), with m the column means of the resident S.
int b2_residual_moments(b2_ctx* ctx, const void* X, int x_dtype, const float* y, int64_t n_rows, int d, int64_t ldx,
                        int mem_kind, const uint8_t* row_mask, int mask_keep, const double* coef, double intercept,
                        int fit_intercept, double* out) {
  if (int r = use_device(ctx)) return r;
  if (int r = check_shape(x_dtype, n_rows, d, ldx, mem_kind)) return r;
  if (coef == nullptr || out == nullptr) { set_error("coef / out is null"); return B2_E_ARG; }
  if (n_rows > 0 && (X == nullptr || y == nullptr)) { set_error("X / y is null"); return B2_E_ARG; }
  if (ctx->n_ranks > 1) {
    set_error("b2_residual_moments runs on one rank only (the residual moments are not exchanged between ranks)");
    return B2_E_UNSUPPORTED;
  }
  if (ctx->d != d) { set_error("the resident statistic has %d features, the rows %d", ctx->d, d); return B2_E_STATE; }
  if (int r = load_refine_state(ctx, d, coef, fit_intercept, &intercept)) return r;
  if (int r = grad_pass(ctx, X, x_dtype, y, n_rows, d, ldx, mem_kind, row_mask, mask_keep)) return r;
  double g[kGradOut];
  B2_CUDA(cudaMemcpyAsync(g, ctx->refine + kRfGrad, sizeof(g), cudaMemcpyDeviceToHost, ctx->stream));
  B2_CUDA(cudaStreamSynchronize(ctx->stream));
  memcpy(out, g, sizeof(double) * d);
  out[d] = g[kMaxD];
  out[d + 1] = g[kMaxD + 1];
  return B2_OK;
}

// The checks both solves share: hyper-parameters finite and >= 0, max_iter >= 1, tol >= 0, outputs present, and the rows
// of the resident S (returned in n)
static int check_bayes_args(b2_ctx* ctx, const double* hyper, int n_hyper, int max_iter, double tol, const double* coef,
                            const double* intercept, const double* alpha_out, const void* lambda_out,
                            const int* n_iter_out, double* n) {
  if (ctx->d == 0) { set_error("b2_gram_reset has not been called"); return B2_E_STATE; }
  if (hyper == nullptr) { set_error("hyper is null"); return B2_E_ARG; }
  for (int k = 0; k < n_hyper; ++k) {
    const bool init = k >= 4;             // alpha_init / lambda_init: NaN means the default
    if (!(isnan(hyper[k]) && init) && !(isfinite(hyper[k]) && hyper[k] >= 0.0)) {
      set_error("hyper[%d] == %g, must be >= 0 and finite%s", k, hyper[k], init ? " (or NaN for the default)" : "");
      return B2_E_ARG;
    }
  }
  if (max_iter < 1) { set_error("max_iter=%d must be >= 1", max_iter); return B2_E_ARG; }
  if (!(tol >= 0.0)) { set_error("tol must be >= 0"); return B2_E_ARG; }
  if (coef == nullptr || intercept == nullptr || alpha_out == nullptr || lambda_out == nullptr || n_iter_out == nullptr) {
    set_error("coef / intercept / alpha_out / lambda_out / n_iter_out is null");
    return B2_E_ARG;
  }
  if (int r = ensure_s_cleared(ctx)) return r;
  const int d = ctx->d;
  B2_CUDA(cudaMemcpyAsync(n, ctx->S + (size_t)d * (d + 2) + d, sizeof(double), cudaMemcpyDeviceToHost, ctx->stream));
  B2_CUDA(cudaStreamSynchronize(ctx->stream));
  return B2_OK;
}

// ctx->enet as [out kByDoubles | anchor 2 kMaxD + 2 | the ARD Gram kMaxD^2 | scores max_iter + 1]; the anchor uploaded
static int bayes_block(b2_ctx* ctx, const double* anchor, int max_iter, int compute_score, int fit_intercept,
                       BayesArgs* a) {
  const size_t off_anchor = kByDoubles, off_A = off_anchor + 2 * kMaxD + 2, off_scores = off_A + (size_t)kMaxD * kMaxD;
  if (int r = ensure_enet_block(ctx, off_scores + (size_t)max_iter + 1)) return r;
  a->max_iter = max_iter;
  a->compute_score = compute_score ? 1 : 0;
  a->fit_intercept = fit_intercept ? 1 : 0;
  a->out = ctx->enet;
  a->A = ctx->enet + off_A;
  a->scores = ctx->enet + off_scores;
  a->anchor = nullptr;
  if (anchor != nullptr) {
    const int d = ctx->d;
    std::vector<double> h(2 * kMaxD + 2, 0.0);
    memcpy(h.data(), anchor, sizeof(double) * d);
    memcpy(h.data() + kMaxD, anchor + d, sizeof(double) * d);
    h[2 * kMaxD] = anchor[2 * d];
    h[2 * kMaxD + 1] = anchor[2 * d + 1];
    B2_CUDA(cudaMemcpyAsync(ctx->enet + off_anchor, h.data(), sizeof(double) * h.size(), cudaMemcpyHostToDevice,
                            ctx->stream));
    B2_CUDA(cudaStreamSynchronize(ctx->stream));   // h is on this frame's stack
    a->anchor = ctx->enet + off_anchor;
  }
  return B2_OK;
}

// The outputs of either solve; n_lambda: 1 (BayesianRidge: one lambda_) or 0 (ARD: d of them).  Returns B2_E_SINGULAR on the kernel's info.
static int fetch_bayes(b2_ctx* ctx, const BayesArgs& a, int n_lambda, double* coef, double* intercept, double* alpha_out,
                       double* lambda_out, int* n_iter_out, double* scores_out, double* sigma_out) {
  const int d = ctx->d;
  double misc[8];
  B2_CUDA(cudaMemcpyAsync(misc, a.out + kByMisc, sizeof(misc), cudaMemcpyDeviceToHost, ctx->stream));
  B2_CUDA(cudaMemcpyAsync(coef, a.out + kByCoef, sizeof(double) * d, cudaMemcpyDeviceToHost, ctx->stream));
  if (n_lambda == 1) B2_CUDA(cudaMemcpyAsync(lambda_out, a.out + kByMisc + 2, sizeof(double), cudaMemcpyDeviceToHost, ctx->stream));
  else B2_CUDA(cudaMemcpyAsync(lambda_out, a.out + kByLambda, sizeof(double) * d, cudaMemcpyDeviceToHost, ctx->stream));
  if (sigma_out != nullptr)
    B2_CUDA(cudaMemcpyAsync(sigma_out, a.out + kBySigma, sizeof(double) * d * d, cudaMemcpyDeviceToHost, ctx->stream));
  B2_CUDA(cudaStreamSynchronize(ctx->stream));
  if (misc[4] != 0.0) {
    set_error("pivot %d of the factorisation of diag(lambda) + alpha A is not positive", (int)misc[4]);
    return B2_E_SINGULAR;
  }
  *intercept = misc[0];
  *alpha_out = misc[1];
  *n_iter_out = (int)misc[3];
  if (scores_out != nullptr && a.compute_score) {     // BayesianRidge scores once more after the loop, ARD does not
    const int n_scores = *n_iter_out + (n_lambda == 1 ? 1 : 0);
    B2_CUDA(cudaMemcpyAsync(scores_out, a.scores, sizeof(double) * n_scores, cudaMemcpyDeviceToHost, ctx->stream));
    B2_CUDA(cudaStreamSynchronize(ctx->stream));
  }
  return B2_OK;
}

int b2_solve_bayes_ridge(b2_ctx* ctx, int fit_intercept, const double* hyper, int max_iter, double tol,
                         const double* anchor, int compute_score, double* coef, double* intercept, double* alpha_out,
                         double* lambda_out, int* n_iter_out, double* scores_out, double* sigma_out) {
  if (int r = use_device(ctx)) return r;
  double n = 0.0;
  if (int r = check_bayes_args(ctx, hyper, 6, max_iter, tol, coef, intercept, alpha_out, lambda_out, n_iter_out, &n))
    return r;
  if (!(n > 0.0)) { set_error("no row kept: the statistic holds no rows"); return B2_E_ARG; }
  BayesArgs a;
  a.a1 = hyper[0]; a.a2 = hyper[1]; a.l1 = hyper[2]; a.l2 = hyper[3]; a.alpha_init = hyper[4]; a.lambda_init = hyper[5];
  a.threshold_lambda = 0.0;
  a.tol = tol;
  if (int r = bayes_block(ctx, anchor, max_iter, compute_score, fit_intercept, &a)) return r;
  if (int r = launch_solve_eigh(ctx, fit_intercept)) return r;
  if (int r = launch_bayes_ridge(ctx, a)) return r;
  double converged = 0.0;
  B2_CUDA(cudaMemcpyAsync(&converged, ctx->loo + kLooMisc + 3, sizeof(double), cudaMemcpyDeviceToHost, ctx->stream));
  if (int r = fetch_bayes(ctx, a, 1, coef, intercept, alpha_out, lambda_out, n_iter_out, scores_out, sigma_out)) return r;
  return eigh_converged(converged);
}

int b2_solve_ard(b2_ctx* ctx, int fit_intercept, const double* hyper, double threshold_lambda, int max_iter, double tol,
                 const double* anchor, int compute_score, double* coef, double* intercept, double* alpha_out,
                 double* lambda_out, int* n_iter_out, double* scores_out, double* sigma_out) {
  if (int r = use_device(ctx)) return r;
  double n = 0.0;
  if (int r = check_bayes_args(ctx, hyper, 4, max_iter, tol, coef, intercept, alpha_out, lambda_out, n_iter_out, &n))
    return r;
  if (!(threshold_lambda >= 0.0)) { set_error("threshold_lambda=%g must be >= 0", threshold_lambda); return B2_E_ARG; }
  if (!(n >= 2.0)) { set_error("the statistic holds %.0f rows, ARDRegression needs at least 2", n); return B2_E_ARG; }
  BayesArgs a;
  a.a1 = hyper[0]; a.a2 = hyper[1]; a.l1 = hyper[2]; a.l2 = hyper[3]; a.alpha_init = NAN; a.lambda_init = NAN;
  a.threshold_lambda = threshold_lambda;
  a.tol = tol;
  if (int r = bayes_block(ctx, anchor, max_iter, compute_score, fit_intercept, &a)) return r;
  if (int r = launch_ard(ctx, a)) return r;
  return fetch_bayes(ctx, a, 0, coef, intercept, alpha_out, lambda_out, n_iter_out, scores_out, sigma_out);
}

// The operands into ctx->enet, then the pass; host rows re-stream through the staging ring, their outputs through two
// device blocks of stage_rows x 2 doubles.
int b2_score_std(b2_ctx* ctx, const void* X, int x_dtype, int64_t n_rows, int d, int64_t ldx, int mem_kind,
                 const double* mean, const double* sigma, double noise_var, const double* coef, double intercept,
                 double* yhat, double* ystd) {
  if (int r = use_device(ctx)) return r;
  if (int r = check_shape(x_dtype, n_rows, d, ldx, mem_kind)) return r;
  if (sigma == nullptr || coef == nullptr || ystd == nullptr) { set_error("sigma / coef / ystd is null"); return B2_E_ARG; }
  if (n_rows > 0 && X == nullptr) { set_error("X is null"); return B2_E_ARG; }
  if (!(noise_var >= 0.0) || !isfinite(noise_var)) { set_error("noise_var=%g must be >= 0 and finite", noise_var); return B2_E_ARG; }
  if (n_rows == 0) return B2_OK;
  if (int r = ensure_enet_block(ctx, kStdDoubles)) return r;
  std::vector<double> op(kStdDoubles, 0.0);
  memcpy(op.data() + kStdSigma, sigma, sizeof(double) * d * d);
  double b_eff = intercept;
  for (int j = 0; j < d; ++j) {
    op[kStdMean + j] = mean != nullptr ? mean[j] : 0.0;
    op[kStdCoef + j] = coef[j];
    b_eff += op[kStdMean + j] * coef[j];
  }
  op[kStdMisc] = b_eff;
  op[kStdMisc + 1] = noise_var;
  B2_CUDA(cudaMemcpyAsync(ctx->enet, op.data(), sizeof(double) * kStdDoubles, cudaMemcpyHostToDevice, ctx->stream));
  if (int r = row_pass(
          ctx, X, x_dtype, nullptr, n_rows, d, ldx, mem_kind, nullptr,
          [&](const RowSpan& s, void* sd, void* yd, void*) {
            return launch_score_std(ctx, s.X, x_dtype, s.rows, d, s.ldx, static_cast<double*>(yd),
                                    static_cast<double*>(sd));
          },
          RowOut{ystd, sizeof(double)}, RowOut{yhat, sizeof(double)}))
    return r;
  B2_CUDA(cudaStreamSynchronize(ctx->stream));     // op is on this frame's stack
  return B2_OK;
}

// ---- PoissonRegressor / GammaRegressor / TweedieRegressor (DESIGN.md section 10) --------------------------------------
// The sums and operands (ctx->glm) and the per-CTA partials (ctx->glm_part), allocated by the first call and freed with
// the context.
static int ensure_glm(b2_ctx* ctx) {
  if (ctx->glm != nullptr) return B2_OK;
  B2_CUDA(cudaMalloc(reinterpret_cast<void**>(&ctx->glm), sizeof(double) * kGlmDoubles));
  B2_CUDA(cudaMalloc(reinterpret_cast<void**>(&ctx->glm_part), sizeof(double) * 2 * (size_t)ctx->sm_count * kGlmPart));
  return B2_OK;
}

// The checks the GLM and logistic entry points share, then the operands (w, step, b, db, the two labels) into ctx->glm
static int glm_operands(b2_ctx* ctx, int x_dtype, int64_t n_rows, int d, int64_t ldx, int mem_kind, const void* X,
                        const float* y, bool need_y, const double* coef, double intercept, const double* step,
                        double step_intercept, double neg_label, double pos_label) {
  if (int r = check_shape(x_dtype, n_rows, d, ldx, mem_kind)) return r;
  if (coef == nullptr) { set_error("coef is null"); return B2_E_ARG; }
  if (n_rows > 0 && (X == nullptr || (need_y && y == nullptr))) { set_error("X / y is null"); return B2_E_ARG; }
  if (ctx->n_ranks > 1) {
    set_error("the GLM passes run on one rank only (their sums are not exchanged between ranks)");
    return B2_E_UNSUPPORTED;
  }
  if (int r = ensure_glm(ctx)) return r;
  std::vector<double> op(2 * kMaxD + 8, 0.0);
  memcpy(op.data() + kGlmOpW, coef, sizeof(double) * d);
  if (step != nullptr) memcpy(op.data() + kGlmOpStep, step, sizeof(double) * d);
  op[kGlmOpMisc] = intercept;
  op[kGlmOpMisc + 1] = step_intercept;
  op[kGlmOpMisc + 2] = neg_label;
  op[kGlmOpMisc + 3] = pos_label;
  B2_CUDA(cudaMemcpyAsync(ctx->glm + kGlmOp, op.data(), sizeof(double) * op.size(), cudaMemcpyHostToDevice, ctx->stream));
  B2_CUDA(cudaStreamSynchronize(ctx->stream));     // op is on this frame's stack
  return B2_OK;
}

static int glm_setup(b2_ctx* ctx, int x_dtype, int64_t n_rows, int d, int64_t ldx, int mem_kind, const void* X,
                     const float* y, bool need_y, int link, double power, const double* coef, double intercept,
                     const double* step, double step_intercept) {
  if (int r = check_shape(x_dtype, n_rows, d, ldx, mem_kind)) return r;
  if (link != B2_GLM_LOG && link != B2_GLM_IDENTITY) { set_error("link=%d must be B2_GLM_LOG or B2_GLM_IDENTITY", link); return B2_E_ARG; }
  if (!isfinite(power)) { set_error("power=%g must be finite", power); return B2_E_ARG; }
  if (link == B2_GLM_IDENTITY && power != 0.0) {
    set_error("the identity link is supported at power 0 only (got power=%g)", power);
    return B2_E_ARG;
  }
  return glm_operands(ctx, x_dtype, n_rows, d, ldx, mem_kind, X, y, need_y, coef, intercept, step, step_intercept, 0.0,
                      0.0);
}

// One pass over the rows into ctx->glm (the first rows overwrite the sums, the others add to them)
static int glm_rows(b2_ctx* ctx, const void* X, int x_dtype, const float* y, int64_t n_rows, int d, int64_t ldx,
                    int mem_kind, const uint8_t* row_mask, int mask_keep, int mode, int family, int link, double power,
                    int n_steps) {
  return row_pass(ctx, X, x_dtype, y, n_rows, d, ldx, mem_kind, row_mask, [&](const RowSpan& s, void*, void*, void*) {
    return launch_glm(ctx, s.X, x_dtype, s.rows, d, s.ldx, s.y, s.mask, mask_keep, mode, family, link, power, n_steps,
                      s.first);
  });
}

// The full symmetric n x n matrix dst from the upper triangle of src (row pitch src_pitch): the upper-block sums of
// b2_dmma.cuh
static void unpack_upper(const double* src, size_t src_pitch, int n, double* dst) {
  for (int i = 0; i < n; ++i)
    for (int j = i; j < n; ++j) dst[(size_t)i * n + j] = dst[(size_t)j * n + i] = src[i * src_pitch + j];
}

// The sums of the last pass (and the mirrored Hessian when hess_out is not null) to the host: [0, 7) and the gradient
// [7, 8 + d), then the extra scalars at 8 + d
static int fetch_glm_sums(b2_ctx* ctx, int d, int n_extra, double* sums_out, double* hess_out) {
  const int d1 = d + 1;
  std::vector<double> h(hess_out != nullptr ? (size_t)kGlmPart : (size_t)kGlmHess);
  B2_CUDA(cudaMemcpyAsync(h.data(), ctx->glm, sizeof(double) * h.size(), cudaMemcpyDeviceToHost, ctx->stream));
  B2_CUDA(cudaStreamSynchronize(ctx->stream));
  memcpy(sums_out, h.data(), sizeof(double) * 7);
  memcpy(sums_out + 7, h.data() + kGlmGrad, sizeof(double) * d1);
  if (n_extra > 0) sums_out[8 + d] = h[kGlmCorrect];
  if (hess_out != nullptr) unpack_upper(h.data() + kGlmHess, kGlmHp, d1, hess_out);
  return B2_OK;
}

int b2_glm_pass(b2_ctx* ctx, const void* X, int x_dtype, const float* y, int64_t n_rows, int d, int64_t ldx,
                int mem_kind, const uint8_t* row_mask, int mask_keep, int link, double power, const double* coef,
                double intercept, int fit_intercept, double* sums_out, double* hess_out) {
  if (int r = use_device(ctx)) return r;
  if (sums_out == nullptr) { set_error("sums_out is null"); return B2_E_ARG; }
  if (int r = glm_setup(ctx, x_dtype, n_rows, d, ldx, mem_kind, X, y, true, link, power, coef,
                        fit_intercept ? intercept : 0.0, nullptr, 0.0))
    return r;
  const int mode = hess_out != nullptr ? kGlmHessian : kGlmGradient;
  if (int r = glm_rows(ctx, X, x_dtype, y, n_rows, d, ldx, mem_kind, row_mask, mask_keep, mode, kGlmTweedie, link, power,
                       0))
    return r;
  return fetch_glm_sums(ctx, d, 0, sums_out, hess_out);
}

int b2_glm_line_search(b2_ctx* ctx, const void* X, int x_dtype, const float* y, int64_t n_rows, int d, int64_t ldx,
                       int mem_kind, const uint8_t* row_mask, int mask_keep, int link, double power, const double* coef,
                       double intercept, const double* step, double step_intercept, int n_steps, double* loss_out) {
  if (int r = use_device(ctx)) return r;
  if (step == nullptr || loss_out == nullptr) { set_error("step / loss_out is null"); return B2_E_ARG; }
  if (n_steps < 1 || n_steps > kGlmSteps) { set_error("n_steps=%d out of range [1,%d]", n_steps, kGlmSteps); return B2_E_ARG; }
  if (int r = glm_setup(ctx, x_dtype, n_rows, d, ldx, mem_kind, X, y, true, link, power, coef, intercept, step,
                        step_intercept))
    return r;
  if (int r = glm_rows(ctx, X, x_dtype, y, n_rows, d, ldx, mem_kind, row_mask, mask_keep, kGlmLadder, kGlmTweedie, link,
                       power, n_steps))
    return r;
  B2_CUDA(cudaMemcpyAsync(loss_out, ctx->glm, sizeof(double) * n_steps, cudaMemcpyDeviceToHost, ctx->stream));
  B2_CUDA(cudaStreamSynchronize(ctx->stream));
  return B2_OK;
}

int b2_glm_predict(b2_ctx* ctx, const void* X, int x_dtype, int64_t n_rows, int d, int64_t ldx, int mem_kind, int link,
                   const double* coef, double intercept, double* mu_out) {
  if (int r = use_device(ctx)) return r;
  if (mu_out == nullptr) { set_error("mu_out is null"); return B2_E_ARG; }
  if (int r = glm_setup(ctx, x_dtype, n_rows, d, ldx, mem_kind, X, nullptr, false, link, 0.0, coef, intercept, nullptr,
                        0.0))
    return r;
  if (n_rows == 0) return B2_OK;
  if (int r = row_pass(
          ctx, X, x_dtype, nullptr, n_rows, d, ldx, mem_kind, nullptr,
          [&](const RowSpan& s, void* mu, void*, void*) {
            return launch_glm_predict(ctx, s.X, x_dtype, s.rows, d, s.ldx, link, static_cast<double*>(mu));
          },
          RowOut{mu_out, sizeof(double)}))
    return r;
  B2_CUDA(cudaStreamSynchronize(ctx->stream));
  return B2_OK;
}

// ---- LogisticRegression (DESIGN.md section 11) ----------------------------------------------------------------------
// The labels are fp32 values: finite, distinct and exactly representable in fp32
static int check_labels(double neg_label, double pos_label) {
  if (!isfinite(neg_label) || !isfinite(pos_label) || (double)(float)neg_label != neg_label ||
      (double)(float)pos_label != pos_label || neg_label == pos_label) {
    set_error("neg_label=%g / pos_label=%g must be two distinct finite fp32 values", neg_label, pos_label);
    return B2_E_ARG;
  }
  return B2_OK;
}

int b2_logistic_pass(b2_ctx* ctx, const void* X, int x_dtype, const float* y, int64_t n_rows, int d, int64_t ldx,
                     int mem_kind, const uint8_t* row_mask, int mask_keep, double neg_label, double pos_label,
                     const double* coef, double intercept, int fit_intercept, double* sums_out, double* hess_out) {
  if (int r = use_device(ctx)) return r;
  if (sums_out == nullptr) { set_error("sums_out is null"); return B2_E_ARG; }
  if (int r = check_labels(neg_label, pos_label)) return r;
  if (int r = glm_operands(ctx, x_dtype, n_rows, d, ldx, mem_kind, X, y, true, coef, fit_intercept ? intercept : 0.0,
                           nullptr, 0.0, neg_label, pos_label))
    return r;
  const int mode = hess_out != nullptr ? kGlmHessian : kGlmGradient;
  if (int r = glm_rows(ctx, X, x_dtype, y, n_rows, d, ldx, mem_kind, row_mask, mask_keep, mode, kGlmBinomial, 0, 0.0, 0))
    return r;
  return fetch_glm_sums(ctx, d, 1, sums_out, hess_out);
}

int b2_logistic_line_search(b2_ctx* ctx, const void* X, int x_dtype, const float* y, int64_t n_rows, int d,
                            int64_t ldx, int mem_kind, const uint8_t* row_mask, int mask_keep, double neg_label,
                            double pos_label, const double* coef, double intercept, const double* step,
                            double step_intercept, int n_steps, double* loss_out) {
  if (int r = use_device(ctx)) return r;
  if (step == nullptr || loss_out == nullptr) { set_error("step / loss_out is null"); return B2_E_ARG; }
  if (n_steps < 1 || n_steps > kGlmSteps) { set_error("n_steps=%d out of range [1,%d]", n_steps, kGlmSteps); return B2_E_ARG; }
  if (int r = check_labels(neg_label, pos_label)) return r;
  if (int r = glm_operands(ctx, x_dtype, n_rows, d, ldx, mem_kind, X, y, true, coef, intercept, step, step_intercept,
                           neg_label, pos_label))
    return r;
  if (int r = glm_rows(ctx, X, x_dtype, y, n_rows, d, ldx, mem_kind, row_mask, mask_keep, kGlmLadder, kGlmBinomial, 0,
                       0.0, n_steps))
    return r;
  B2_CUDA(cudaMemcpyAsync(loss_out, ctx->glm, sizeof(double) * n_steps, cudaMemcpyDeviceToHost, ctx->stream));
  B2_CUDA(cudaStreamSynchronize(ctx->stream));
  return B2_OK;
}

int b2_logistic_predict(b2_ctx* ctx, const void* X, int x_dtype, int64_t n_rows, int d, int64_t ldx, int mem_kind,
                        const double* coef, double intercept, double neg_label, double pos_label, double* decision_out,
                        double* proba_out, float* label_out) {
  if (int r = use_device(ctx)) return r;
  if (decision_out == nullptr && proba_out == nullptr && label_out == nullptr) {
    set_error("decision_out, proba_out and label_out are all null");
    return B2_E_ARG;
  }
  if (int r = check_labels(neg_label, pos_label)) return r;
  if (int r = glm_operands(ctx, x_dtype, n_rows, d, ldx, mem_kind, X, nullptr, false, coef, intercept, nullptr, 0.0,
                           neg_label, pos_label))
    return r;
  if (n_rows == 0) return B2_OK;
  if (int r = row_pass(
          ctx, X, x_dtype, nullptr, n_rows, d, ldx, mem_kind, nullptr,
          [&](const RowSpan& s, void* dec, void* pr, void* lab) {
            return launch_logistic_predict(ctx, s.X, x_dtype, s.rows, d, s.ldx, static_cast<double*>(dec),
                                           static_cast<double*>(pr), static_cast<float*>(lab));
          },
          RowOut{decision_out, sizeof(double)}, RowOut{proba_out, 2 * sizeof(double)},
          RowOut{label_out, sizeof(float)}))
    return r;
  B2_CUDA(cudaStreamSynchronize(ctx->stream));
  return B2_OK;
}

int b2_label_scan(b2_ctx* ctx, const float* y, int64_t n_rows, const uint8_t* row_mask, int mask_keep,
                  double* stats_out) {
  if (int r = use_device(ctx)) return r;
  if (stats_out == nullptr) { set_error("stats_out is null"); return B2_E_ARG; }
  if (n_rows < 0 || (n_rows > 0 && y == nullptr)) { set_error("n_rows=%lld / y is null", (long long)n_rows); return B2_E_ARG; }
  if (ctx->n_ranks > 1) {
    set_error("the label scan runs on one rank only (its counts are not exchanged between ranks)");
    return B2_E_UNSUPPORTED;
  }
  if (int r = ensure_glm(ctx)) return r;
  unsigned long long* st = reinterpret_cast<unsigned long long*>(ctx->glm_part);
  if (int r = launch_label_scan(ctx, y, n_rows, row_mask, mask_keep, st)) return r;
  unsigned long long h[kLabelWords];
  B2_CUDA(cudaMemcpyAsync(h, st, sizeof(h), cudaMemcpyDeviceToHost, ctx->stream));
  B2_CUDA(cudaStreamSynchronize(ctx->stream));
  const bool any = h[kLabelMin] <= h[kLabelMax];     // some kept y is finite
  auto value = [](unsigned long long k) {            // the inverse of the kernel's order-preserving key
    uint32_t u = (uint32_t)k;
    u = (u & 0x80000000u) ? (u & 0x7fffffffu) : ~u;
    float f;
    memcpy(&f, &u, sizeof(f));
    return (double)f;
  };
  stats_out[0] = (double)h[kLabelKept];
  stats_out[1] = (double)h[kLabelNonFinite];
  stats_out[2] = (double)h[kLabelNonIntegral];
  stats_out[3] = any ? value(h[kLabelMin]) : NAN;
  stats_out[4] = any ? value(h[kLabelMax]) : NAN;
  stats_out[5] = (double)h[kLabelNMin];
  stats_out[6] = (double)h[kLabelNMax];
  return B2_OK;
}

// ---- RidgeClassifier (DESIGN.md section 12) ------------------------------------------------------------------------
// The operands and sums (ctx->cls) beside the GLM block, whose per-CTA partials the passes share; allocated by the first
// call and freed with the context.
static int ensure_cls(b2_ctx* ctx, const char* what) {
  if (ctx->n_ranks > 1) {
    set_error("%s runs on one rank only (its sums are not exchanged between ranks)", what);
    return B2_E_UNSUPPORTED;
  }
  if (int r = ensure_glm(ctx)) return r;
  if (ctx->cls == nullptr) B2_CUDA(cudaMalloc(reinterpret_cast<void**>(&ctx->cls), sizeof(double) * kClsDoubles));
  return B2_OK;
}

// n_classes sorted, distinct, finite fp32 values, 2 <= n_classes <= B2_MAX_CLASSES
static int check_classes(const float* classes, int n_classes) {
  if (classes == nullptr || n_classes < 2 || n_classes > kMaxClasses) {
    set_error("classes: 2..%d sorted fp32 values expected (got %d%s)", kMaxClasses, n_classes,
              classes == nullptr ? ", null" : "");
    return B2_E_ARG;
  }
  for (int k = 0; k < n_classes; ++k)
    if (!isfinite(classes[k]) || (k > 0 && !(classes[k] > classes[k - 1]))) {
      set_error("classes must be finite and strictly ascending (class %d is %g)", k, (double)classes[k]);
      return B2_E_ARG;
    }
  return B2_OK;
}

// doubles [at, at + n) of ctx->cls from the host
static int upload_cls(b2_ctx* ctx, int at, const std::vector<double>& v) {
  B2_CUDA(cudaMemcpyAsync(ctx->cls + at, v.data(), sizeof(double) * v.size(), cudaMemcpyHostToDevice, ctx->stream));
  B2_CUDA(cudaStreamSynchronize(ctx->stream));     // v belongs to the caller's frame
  return B2_OK;
}

int b2_class_sums(b2_ctx* ctx, const void* X, int x_dtype, const float* y, int64_t n_rows, int d, int64_t ldx,
                  int mem_kind, const uint8_t* row_mask, int mask_keep, const float* classes, int n_classes,
                  const double* center, double* sums_out, double* counts_out) {
  if (int r = use_device(ctx)) return r;
  if (int r = check_shape(x_dtype, n_rows, d, ldx, mem_kind)) return r;
  if (n_rows > 0 && (X == nullptr || y == nullptr)) { set_error("X / y is null"); return B2_E_ARG; }
  if (sums_out == nullptr || counts_out == nullptr) { set_error("sums_out / counts_out is null"); return B2_E_ARG; }
  if (int r = check_classes(classes, n_classes)) return r;
  if (int r = ensure_cls(ctx, "b2_class_sums")) return r;
  std::vector<double> op(kMaxD + kMaxClasses, 0.0);     // kClsCenter, then kClsClasses
  if (center != nullptr) memcpy(op.data() + kClsCenter, center, sizeof(double) * d);
  for (int k = 0; k < n_classes; ++k) op[kClsClasses + k] = classes[k];
  if (int r = upload_cls(ctx, kClsCenter, op)) return r;
  if (int r = row_pass(ctx, X, x_dtype, y, n_rows, d, ldx, mem_kind, row_mask, [&](const RowSpan& s, void*, void*, void*) {
        return launch_class_sums(ctx, s.X, x_dtype, s.rows, d, s.ldx, s.y, s.mask, mask_keep, n_classes, s.first);
      }))
    return r;
  const int n_sums = n_classes * (d + 1);
  std::vector<double> h((size_t)n_sums + 3);
  B2_CUDA(cudaMemcpyAsync(h.data(), ctx->cls + kClsSums, sizeof(double) * h.size(), cudaMemcpyDeviceToHost, ctx->stream));
  B2_CUDA(cudaStreamSynchronize(ctx->stream));
  memcpy(sums_out, h.data(), sizeof(double) * n_sums);
  memcpy(counts_out, h.data() + n_sums, sizeof(double) * 3);
  return B2_OK;
}

// ---- LinearDiscriminantAnalysis (DESIGN.md section 16) ---------------------------------------------------------------
// The operands and sums (ctx->disc) and the per-CTA partials (ctx->disc_part, one CTA per SM), allocated by the first
// call and freed with the context: no other pass's buffers are touched.
int b2_class_scatter(b2_ctx* ctx, const void* X, int x_dtype, const float* y, int64_t n_rows, int d, int64_t ldx,
                     int mem_kind, const uint8_t* row_mask, int mask_keep, const float* classes, int n_classes,
                     const double* means, const double* weights, double* scatter_out, double* counts_out) {
  if (int r = use_device(ctx)) return r;
  if (int r = check_shape(x_dtype, n_rows, d, ldx, mem_kind)) return r;
  if (n_rows > 0 && (X == nullptr || y == nullptr)) { set_error("X / y is null"); return B2_E_ARG; }
  if (means == nullptr || scatter_out == nullptr || counts_out == nullptr) {
    set_error("means / scatter_out / counts_out is null");
    return B2_E_ARG;
  }
  if (int r = check_classes(classes, n_classes)) return r;
  std::vector<double> op(kDaSums, 0.0);                 // kDaClasses, kDaWeights, kDaMeans
  for (int k = 0; k < n_classes; ++k) {
    const double w = weights != nullptr ? weights[k] : 1.0;
    if (!(w >= 0.0) || !isfinite(w)) { set_error("weights[%d]=%g must be finite and >= 0", k, w); return B2_E_ARG; }
    op[kDaClasses + k] = classes[k];
    op[kDaWeights + k] = w;
    for (int j = 0; j < d; ++j) {
      const double m = means[(size_t)k * d + j];
      if (!isfinite(m)) { set_error("means[%d][%d]=%g is not finite", k, j, m); return B2_E_ARG; }
      op[kDaMeans + k * kMaxD + j] = m;
    }
  }
  if (ctx->n_ranks > 1) {
    set_error("b2_class_scatter runs on one rank only (its sums are not exchanged between ranks)");
    return B2_E_UNSUPPORTED;
  }
  if (ctx->disc == nullptr) {
    B2_CUDA(cudaMalloc(reinterpret_cast<void**>(&ctx->disc), sizeof(double) * kDaDoubles));
    B2_CUDA(cudaMalloc(reinterpret_cast<void**>(&ctx->disc_part), sizeof(double) * (size_t)ctx->sm_count * kDaPart));
  }
  B2_CUDA(cudaMemcpyAsync(ctx->disc, op.data(), sizeof(double) * op.size(), cudaMemcpyHostToDevice, ctx->stream));
  B2_CUDA(cudaStreamSynchronize(ctx->stream));     // op is on this frame's stack
  if (int r = row_pass(ctx, X, x_dtype, y, n_rows, d, ldx, mem_kind, row_mask, [&](const RowSpan& s, void*, void*, void*) {
        return launch_class_scatter(ctx, s.X, x_dtype, s.rows, d, s.ldx, s.y, s.mask, mask_keep, n_classes, s.first);
      }))
    return r;
  std::vector<double> h(kDaPart);
  B2_CUDA(cudaMemcpyAsync(h.data(), ctx->disc + kDaSums, sizeof(double) * h.size(), cudaMemcpyDeviceToHost, ctx->stream));
  B2_CUDA(cudaStreamSynchronize(ctx->stream));
  memcpy(counts_out, h.data(), sizeof(double) * 3);
  unpack_upper(h.data() + kDaHead, kMaxD, d, scatter_out);
  return B2_OK;
}

// ---- QuadraticDiscriminantAnalysis (DESIGN.md section 17) -----------------------------------------------------------
// The operands and sums (ctx->qda), the int header (ctx->qda_hd) and the scratch, allocated by the first call and freed
// with the context: no other pass's buffers are touched.  The classes and means (both entry points) into ctx->qda.
static int qda_setup(b2_ctx* ctx, const char* what, const void* X, int x_dtype, int64_t n_rows, int d, int64_t ldx,
                     int mem_kind, const float* classes, int n_classes, const double* means, std::vector<double>& op) {
  if (int r = check_shape(x_dtype, n_rows, d, ldx, mem_kind)) return r;
  if (n_rows > 0 && X == nullptr) { set_error("X is null"); return B2_E_ARG; }
  if (means == nullptr) { set_error("means is null"); return B2_E_ARG; }
  if (int r = check_classes(classes, n_classes)) return r;
  for (int k = 0; k < n_classes; ++k) {
    op[kQdClasses + k] = classes[k];
    for (int j = 0; j < d; ++j) {
      const double m = means[(size_t)k * d + j];
      if (!isfinite(m)) { set_error("means[%d][%d]=%g is not finite", k, j, m); return B2_E_ARG; }
      op[kQdMeans + k * kMaxD + j] = m;
    }
  }
  if (ctx->n_ranks > 1) {
    set_error("%s runs on one rank only (its sums are not exchanged between ranks)", what);
    return B2_E_UNSUPPORTED;
  }
  if (ctx->qda == nullptr) {
    B2_CUDA(cudaMalloc(reinterpret_cast<void**>(&ctx->qda), sizeof(double) * kQdDoubles));
    B2_CUDA(cudaMalloc(reinterpret_cast<void**>(&ctx->qda_hd), sizeof(int) * (kQdHdItems + 3 * (size_t)qda_max_items(ctx))));
    B2_CUDA(cudaMalloc(&ctx->qda_scratch, kQdScratchBytes));
  }
  B2_CUDA(cudaMemcpyAsync(ctx->qda, op.data(), sizeof(double) * op.size(), cudaMemcpyHostToDevice, ctx->stream));
  B2_CUDA(cudaStreamSynchronize(ctx->stream));     // op is on the caller's stack
  return B2_OK;
}

int b2_class_scatters(b2_ctx* ctx, const void* X, int x_dtype, const float* y, int64_t n_rows, int d, int64_t ldx,
                      int mem_kind, const uint8_t* row_mask, int mask_keep, const float* classes, int n_classes,
                      const double* means, double* scatters_out, double* class_counts_out, double* counts_out) {
  if (int r = use_device(ctx)) return r;
  if (n_rows > 0 && y == nullptr) { set_error("y is null"); return B2_E_ARG; }
  if (scatters_out == nullptr || class_counts_out == nullptr || counts_out == nullptr) {
    set_error("scatters_out / class_counts_out / counts_out is null");
    return B2_E_ARG;
  }
  std::vector<double> op(kQdConst, 0.0);                 // kQdClasses, kQdMeans
  if (int r = qda_setup(ctx, "b2_class_scatters", X, x_dtype, n_rows, d, ldx, mem_kind, classes, n_classes, means, op))
    return r;
  if (ctx->qda_part == nullptr)
    B2_CUDA(cudaMalloc(reinterpret_cast<void**>(&ctx->qda_part),
                       sizeof(double) * (size_t)qda_max_items(ctx) * kMaxD * kMaxD));
  // device rows in spans of at most kQdSpan rows (host blocks are shorter), the sums accumulating across them
  if (int r = row_pass(ctx, X, x_dtype, y, n_rows, d, ldx, mem_kind, row_mask, [&](const RowSpan& s, void*, void*, void*) {
        const int es = x_dtype == B2_F32 ? 4 : 2;
        for (int64_t r0 = 0; r0 < s.rows || (r0 == 0 && s.first); r0 += kQdSpan) {
          const int64_t rows = s.rows - r0 < kQdSpan ? s.rows - r0 : kQdSpan;
          const void* Xs = static_cast<const char*>(s.X) + (size_t)r0 * s.ldx * es;
          if (int rc = launch_class_scatters(ctx, Xs, x_dtype, rows, d, s.ldx, s.y != nullptr ? s.y + r0 : nullptr,
                                             s.mask != nullptr ? s.mask + r0 : nullptr, mask_keep, n_classes,
                                             s.first && r0 == 0))
            return rc;
          if (rows == 0) break;
        }
        return (int)B2_OK;
      }))
    return r;
  std::vector<double> h((size_t)n_classes * kMaxD * kMaxD);
  B2_CUDA(cudaMemcpyAsync(h.data(), ctx->qda + kQdSums, sizeof(double) * h.size(), cudaMemcpyDeviceToHost, ctx->stream));
  double c[kMaxClasses + 3];
  B2_CUDA(cudaMemcpyAsync(c, ctx->qda + kQdCounts, sizeof(c), cudaMemcpyDeviceToHost, ctx->stream));
  B2_CUDA(cudaStreamSynchronize(ctx->stream));
  for (int k = 0; k < n_classes; ++k) {
    class_counts_out[k] = c[k];
    unpack_upper(h.data() + (size_t)k * kMaxD * kMaxD, kMaxD, d, scatters_out + (size_t)k * d * d);
  }
  memcpy(counts_out, c + kMaxClasses, sizeof(double) * 3);
  return B2_OK;
}

int b2_qda_decision(b2_ctx* ctx, const void* X, int x_dtype, const float* y, int64_t n_rows, int d, int64_t ldx,
                    int mem_kind, const uint8_t* row_mask, int mask_keep, const float* classes, int n_classes,
                    const double* means, const double* transforms, const double* offsets, double* decision_out,
                    float* label_out, double* diff_out, double* counts_out) {
  if (int r = use_device(ctx)) return r;
  if (transforms == nullptr || offsets == nullptr) { set_error("transforms / offsets is null"); return B2_E_ARG; }
  if (decision_out == nullptr && label_out == nullptr && diff_out == nullptr && counts_out == nullptr) {
    set_error("decision_out, label_out, diff_out and counts_out are all null");
    return B2_E_ARG;
  }
  if (n_rows > 0 && counts_out != nullptr && y == nullptr) { set_error("counts_out needs y"); return B2_E_ARG; }
  if (diff_out != nullptr && n_classes != 2) { set_error("diff_out needs two classes (got %d)", n_classes); return B2_E_ARG; }
  if (n_classes < 2 || n_classes > kMaxClasses) return check_classes(classes, n_classes);
  std::vector<double> op(kQdW + (size_t)n_classes * d * d, 0.0);   // kQdClasses, kQdMeans, kQdConst, kQdW (pitch d)
  for (int k = 0; k < n_classes; ++k) {
    if (!isfinite(offsets[k])) { set_error("offsets[%d]=%g is not finite", k, offsets[k]); return B2_E_ARG; }
    op[kQdConst + k] = offsets[k];
  }
  for (size_t e = 0; e < (size_t)n_classes * d * d; ++e) {
    if (!isfinite(transforms[e])) { set_error("transforms[%zu]=%g is not finite", e, transforms[e]); return B2_E_ARG; }
    op[kQdW + e] = transforms[e];
  }
  if (int r = qda_setup(ctx, "b2_qda_decision", X, x_dtype, n_rows, d, ldx, mem_kind, classes, n_classes, means, op))
    return r;
  if (counts_out != nullptr)
    B2_CUDA(cudaMemsetAsync(ctx->qda_hd + kQdHdCorrect, 0, 2 * sizeof(unsigned long long), ctx->stream));
  // y and the mask only count: every row gets its decision and label
  const float* yc = counts_out != nullptr ? y : nullptr;
  const uint8_t* mc = counts_out != nullptr ? row_mask : nullptr;
  if (int r = row_pass(
          ctx, X, x_dtype, yc, n_rows, d, ldx, mem_kind, mc,
          [&](const RowSpan& s, void* dec, void* lab, void* dif) {
            if (dec != nullptr)
              return launch_qda_decision(ctx, s.X, x_dtype, s.rows, d, s.ldx, s.y, s.mask, mask_keep, n_classes,
                                         static_cast<double*>(dec), static_cast<float*>(lab), static_cast<double*>(dif));
            // no decisions wanted: they go through the scratch, in parts that fit it
            const int64_t part = (int64_t)(kQdScratchBytes / sizeof(double)) / n_classes;
            const int es = x_dtype == B2_F32 ? 4 : 2;
            for (int64_t r0 = 0; r0 < s.rows; r0 += part) {
              const int64_t rows = s.rows - r0 < part ? s.rows - r0 : part;
              if (int rc = launch_qda_decision(ctx, static_cast<const char*>(s.X) + (size_t)r0 * s.ldx * es, x_dtype,
                                               rows, d, s.ldx, s.y != nullptr ? s.y + r0 : nullptr,
                                               s.mask != nullptr ? s.mask + r0 : nullptr, mask_keep, n_classes,
                                               static_cast<double*>(ctx->qda_scratch),
                                               lab != nullptr ? static_cast<float*>(lab) + r0 : nullptr,
                                               dif != nullptr ? static_cast<double*>(dif) + r0 : nullptr))
                return rc;
            }
            return (int)B2_OK;
          },
          RowOut{decision_out, sizeof(double) * n_classes}, RowOut{label_out, sizeof(float)},
          RowOut{diff_out, sizeof(double)}))
    return r;
  if (counts_out != nullptr) {
    unsigned long long c[2];
    B2_CUDA(cudaMemcpyAsync(c, ctx->qda_hd + kQdHdCorrect, sizeof(c), cudaMemcpyDeviceToHost, ctx->stream));
    B2_CUDA(cudaStreamSynchronize(ctx->stream));
    counts_out[0] = (double)c[0];
    counts_out[1] = (double)c[1];
  }
  B2_CUDA(cudaStreamSynchronize(ctx->stream));
  return B2_OK;
}

int b2_solve_classes(b2_ctx* ctx, double alpha, int fit_intercept, const double* class_sums, int n_classes,
                     double* coef_out, double* intercept_out) {
  if (int r = use_device(ctx)) return r;
  if (ctx->d == 0) { set_error("b2_gram_reset has not been called"); return B2_E_STATE; }
  if (!(alpha >= 0.0) || !isfinite(alpha)) { set_error("alpha must be finite and >= 0"); return B2_E_ARG; }
  if (n_classes < 2 || n_classes > kMaxClasses) {
    set_error("n_classes=%d out of range [2,%d]", n_classes, kMaxClasses);
    return B2_E_ARG;
  }
  if (coef_out == nullptr || intercept_out == nullptr) { set_error("coef_out / intercept_out is null"); return B2_E_ARG; }
  if (int r = ensure_cls(ctx, "b2_solve_classes")) return r;
  const int d = ctx->d, T = n_classes == 2 ? 1 : n_classes;
  if (class_sums != nullptr) {
    std::vector<double> v(class_sums, class_sums + (size_t)n_classes * (d + 1));
    if (int r = upload_cls(ctx, kClsSums, v)) return r;
  }
  if (int r = ensure_s_cleared(ctx)) return r;
  if (int r = launch_solve_classes(ctx, alpha, fit_intercept, n_classes)) return r;
  std::vector<double> h(kClsInfo + 1 - kClsCoef);       // W, b, info
  B2_CUDA(cudaMemcpyAsync(h.data(), ctx->cls + kClsCoef, sizeof(double) * h.size(), cudaMemcpyDeviceToHost, ctx->stream));
  B2_CUDA(cudaStreamSynchronize(ctx->stream));
  const double info = h[kClsInfo - kClsCoef];
  if (info != 0.0) {
    set_error("pivot %d of the LDL^T factorisation is not positive: the centred Gram matrix is rank deficient "
              "(use alpha > 0 or b2_solve_eigh)", (int)info);
    return B2_E_SINGULAR;
  }
  for (int t = 0; t < T; ++t) {
    memcpy(coef_out + (size_t)t * d, h.data() + (size_t)t * kMaxD, sizeof(double) * d);
    intercept_out[t] = h[kClsIntercept - kClsCoef + t];
  }
  return B2_OK;
}

int b2_classify(b2_ctx* ctx, const void* X, int x_dtype, const float* y, int64_t n_rows, int d, int64_t ldx,
                int mem_kind, const uint8_t* row_mask, int mask_keep, const double* coef, const double* intercept,
                int n_targets, const float* classes, double* decision_out, float* label_out, double* counts_out) {
  if (int r = use_device(ctx)) return r;
  if (int r = check_shape(x_dtype, n_rows, d, ldx, mem_kind)) return r;
  if (n_targets < 1 || n_targets > kMaxClasses) {
    set_error("n_targets=%d out of range [1,%d]", n_targets, kMaxClasses);
    return B2_E_ARG;
  }
  if (coef == nullptr || intercept == nullptr) { set_error("coef / intercept is null"); return B2_E_ARG; }
  if (decision_out == nullptr && label_out == nullptr && counts_out == nullptr) {
    set_error("decision_out, label_out and counts_out are all null");
    return B2_E_ARG;
  }
  if (n_rows > 0 && (X == nullptr || (counts_out != nullptr && y == nullptr))) {
    set_error("X / y is null (counts_out needs y)");
    return B2_E_ARG;
  }
  const int n_classes = n_targets == 1 ? 2 : n_targets;
  if (int r = check_classes(classes, n_classes)) return r;
  if (int r = ensure_cls(ctx, "b2_classify")) return r;
  std::vector<double> op(kClsInfo - kClsClasses, 0.0);  // classes, W, b
  for (int k = 0; k < n_classes; ++k) op[k] = classes[k];
  for (int t = 0; t < n_targets; ++t) {
    memcpy(op.data() + kClsCoef - kClsClasses + (size_t)t * kMaxD, coef + (size_t)t * d, sizeof(double) * d);
    op[kClsIntercept - kClsClasses + t] = intercept[t];
  }
  if (int r = upload_cls(ctx, kClsClasses, op)) return r;
  // y and the mask only count: every row gets its decision and label
  const float* yc = counts_out != nullptr ? y : nullptr;
  const uint8_t* mc = counts_out != nullptr ? row_mask : nullptr;
  if (int r = row_pass(
          ctx, X, x_dtype, yc, n_rows, d, ldx, mem_kind, mc,
          [&](const RowSpan& s, void* dec, void* lab, void*) {
            return launch_classify(ctx, s.X, x_dtype, s.rows, d, s.ldx, s.y, s.mask, mask_keep, n_targets,
                                   static_cast<double*>(dec), static_cast<float*>(lab), s.first);
          },
          RowOut{decision_out, sizeof(double) * n_targets}, RowOut{label_out, sizeof(float)}))
    return r;
  if (counts_out != nullptr)
    B2_CUDA(cudaMemcpyAsync(counts_out, ctx->cls + kClsCounts, sizeof(double) * 2, cudaMemcpyDeviceToHost, ctx->stream));
  B2_CUDA(cudaStreamSynchronize(ctx->stream));
  return B2_OK;
}

int b2_label_values(b2_ctx* ctx, const float* y, int64_t n_rows, const uint8_t* row_mask, int mask_keep,
                    int max_values, float* values_out, int* n_values_out, int* more_out) {
  if (int r = use_device(ctx)) return r;
  if (n_rows < 0 || (n_rows > 0 && y == nullptr)) { set_error("n_rows=%lld / y is null", (long long)n_rows); return B2_E_ARG; }
  if (max_values < 1 || max_values > kMaxClasses) {
    set_error("max_values=%d out of range [1,%d]", max_values, kMaxClasses);
    return B2_E_ARG;
  }
  if (values_out == nullptr || n_values_out == nullptr || more_out == nullptr) {
    set_error("values_out / n_values_out / more_out is null");
    return B2_E_ARG;
  }
  if (int r = ensure_cls(ctx, "b2_label_values")) return r;
  unsigned long long* st = reinterpret_cast<unsigned long long*>(ctx->glm_part);
  if (int r = launch_label_values(ctx, y, n_rows, row_mask, mask_keep, max_values, st)) return r;
  unsigned long long h[kMaxClasses + 1];
  B2_CUDA(cudaMemcpyAsync(h, st, sizeof(unsigned long long) * (max_values + 1), cudaMemcpyDeviceToHost, ctx->stream));
  B2_CUDA(cudaStreamSynchronize(ctx->stream));
  int found = 0;
  for (; found < max_values && h[found] != ~0ull; ++found) {
    uint32_t u = (uint32_t)h[found];                   // the inverse of the kernel's order-preserving key
    u = (u & 0x80000000u) ? (u & 0x7fffffffu) : ~u;
    memcpy(values_out + found, &u, sizeof(float));
  }
  *n_values_out = found;
  *more_out = h[max_values] != ~0ull ? 1 : 0;
  return B2_OK;
}

// ---- multinomial LogisticRegression (DESIGN.md section 14) ---------------------------------------------------------
// The checks the multinomial entry points share, then the classes, coefficients and step (K x (d + 1) each, row k =
// [w_k, b_k]; step may be null) into ctx->mn_op and room for the reduced sums of `mode` in ctx->mn_sum
static int mn_setup(b2_ctx* ctx, const void* X, int x_dtype, const float* y, int64_t n_rows, int d, int64_t ldx,
                    int mem_kind, const float* classes, int n_classes, const double* coef, const double* step,
                    int fit_intercept, int mode) {
  if (int r = check_shape(x_dtype, n_rows, d, ldx, mem_kind)) return r;
  if (n_rows > 0 && (X == nullptr || y == nullptr)) { set_error("X / y is null"); return B2_E_ARG; }
  if (coef == nullptr) { set_error("coef is null"); return B2_E_ARG; }
  if (n_classes < 3 || n_classes > kMaxClasses) {
    set_error("n_classes=%d out of range [3,%d] (two classes: b2_logistic_pass)", n_classes, kMaxClasses);
    return B2_E_ARG;
  }
  if (int r = check_classes(classes, n_classes)) return r;
  if (ctx->n_ranks > 1) {
    set_error("the multinomial passes run on one rank only (their sums are not exchanged between ranks)");
    return B2_E_UNSUPPORTED;
  }
  if (ctx->mn_op == nullptr) B2_CUDA(cudaMalloc(reinterpret_cast<void**>(&ctx->mn_op), sizeof(double) * kMnOpDoubles));
  const size_t sum = multinomial_sum_doubles(d, n_classes, mode);
  if (sum > ctx->mn_sum_doubles) {
    if (ctx->mn_sum != nullptr) cudaFree(ctx->mn_sum);
    ctx->mn_sum = nullptr;
    ctx->mn_sum_doubles = 0;
    B2_CUDA(cudaMalloc(reinterpret_cast<void**>(&ctx->mn_sum), sizeof(double) * sum));
    ctx->mn_sum_doubles = sum;
  }
  std::vector<double> op(kMnOpDoubles, 0.0);
  for (int k = 0; k < n_classes; ++k) {
    op[kMnClasses + k] = classes[k];
    for (int j = 0; j <= d; ++j) {
      const bool w = j < d || fit_intercept;   // the intercept column is zero without fit_intercept
      op[kMnCoef + k * (kMaxD + 1) + j] = w ? coef[(size_t)k * (d + 1) + j] : 0.0;
      if (step != nullptr) op[kMnStep + k * (kMaxD + 1) + j] = w ? step[(size_t)k * (d + 1) + j] : 0.0;
    }
  }
  B2_CUDA(cudaMemcpyAsync(ctx->mn_op, op.data(), sizeof(double) * op.size(), cudaMemcpyHostToDevice, ctx->stream));
  B2_CUDA(cudaStreamSynchronize(ctx->stream));     // op is on this frame's stack
  return B2_OK;
}

static int mn_rows(b2_ctx* ctx, const void* X, int x_dtype, const float* y, int64_t n_rows, int d, int64_t ldx,
                   int mem_kind, const uint8_t* row_mask, int mask_keep, int mode, int n_classes, int n_steps) {
  return row_pass(ctx, X, x_dtype, y, n_rows, d, ldx, mem_kind, row_mask, [&](const RowSpan& s, void*, void*, void*) {
    return launch_multinomial(ctx, s.X, x_dtype, s.rows, d, s.ldx, s.y, s.mask, mask_keep, mode, n_classes, n_steps,
                              s.first);
  });
}

int b2_multinomial_pass(b2_ctx* ctx, const void* X, int x_dtype, const float* y, int64_t n_rows, int d, int64_t ldx,
                        int mem_kind, const uint8_t* row_mask, int mask_keep, const float* classes, int n_classes,
                        const double* coef, int fit_intercept, double* sums_out, double* hess_out) {
  if (int r = use_device(ctx)) return r;
  if (sums_out == nullptr) { set_error("sums_out is null"); return B2_E_ARG; }
  const int mode = hess_out != nullptr ? kGlmHessian : kGlmGradient;
  if (int r = mn_setup(ctx, X, x_dtype, y, n_rows, d, ldx, mem_kind, classes, n_classes, coef, nullptr, fit_intercept,
                       mode))
    return r;
  if (int r = mn_rows(ctx, X, x_dtype, y, n_rows, d, ldx, mem_kind, row_mask, mask_keep, mode, n_classes, 0)) return r;
  const int K = n_classes, d1 = d + 1, dp = (d1 + 15) & ~15;
  std::vector<double> h(multinomial_sum_doubles(d, K, mode));
  B2_CUDA(cudaMemcpyAsync(h.data(), ctx->mn_sum, sizeof(double) * h.size(), cudaMemcpyDeviceToHost, ctx->stream));
  B2_CUDA(cudaStreamSynchronize(ctx->stream));
  memcpy(sums_out, h.data(), sizeof(double) * 5);
  memcpy(sums_out + 5, h.data() + kMnHead, sizeof(double) * K * d1);
  if (hess_out != nullptr) {
    // block (k, l) and block (l, k) are the same symmetric matrix: its upper triangle, mirrored
    const double* blk = h.data() + kMnHead + (size_t)K * d1;
    for (int k = 0, p = 0; k < K; ++k)
      for (int l = k; l < K; ++l, ++p) {
        const double* b = blk + (size_t)p * dp * dp;
        unpack_upper(b, dp, d1, hess_out + ((size_t)k * K + l) * d1 * d1);
        unpack_upper(b, dp, d1, hess_out + ((size_t)l * K + k) * d1 * d1);
      }
  }
  return B2_OK;
}

int b2_multinomial_line_search(b2_ctx* ctx, const void* X, int x_dtype, const float* y, int64_t n_rows, int d,
                               int64_t ldx, int mem_kind, const uint8_t* row_mask, int mask_keep, const float* classes,
                               int n_classes, const double* coef, const double* step, int n_steps, double* loss_out) {
  if (int r = use_device(ctx)) return r;
  if (step == nullptr || loss_out == nullptr) { set_error("step / loss_out is null"); return B2_E_ARG; }
  if (n_steps < 1 || n_steps > kGlmSteps) { set_error("n_steps=%d out of range [1,%d]", n_steps, kGlmSteps); return B2_E_ARG; }
  if (int r = mn_setup(ctx, X, x_dtype, y, n_rows, d, ldx, mem_kind, classes, n_classes, coef, step, 1, kGlmLadder))
    return r;
  if (int r = mn_rows(ctx, X, x_dtype, y, n_rows, d, ldx, mem_kind, row_mask, mask_keep, kGlmLadder, n_classes,
                      n_steps))
    return r;
  B2_CUDA(cudaMemcpyAsync(loss_out, ctx->mn_sum, sizeof(double) * n_steps, cudaMemcpyDeviceToHost, ctx->stream));
  B2_CUDA(cudaStreamSynchronize(ctx->stream));
  return B2_OK;
}

int b2_softmax_rows(b2_ctx* ctx, double* values, int64_t n_rows, int n_cols, int mem_kind) {
  if (int r = use_device(ctx)) return r;
  if (n_rows < 0 || n_cols < 1 || (n_rows > 0 && values == nullptr)) {
    set_error("n_rows=%lld / n_cols=%d / values is null", (long long)n_rows, n_cols);
    return B2_E_ARG;
  }
  if (mem_kind != B2_MEM_DEVICE && mem_kind != B2_MEM_HOST) { set_error("bad mem_kind %d", mem_kind); return B2_E_ARG; }
  if (n_rows == 0) return B2_OK;
  const size_t bytes = sizeof(double) * (size_t)n_rows * n_cols;
  if (mem_kind == B2_MEM_DEVICE) {
    if (int r = launch_softmax_rows(ctx, values, n_rows, n_cols)) return r;
    B2_CUDA(cudaStreamSynchronize(ctx->stream));
    return B2_OK;
  }
  double* dev = nullptr;                            // host values: one round trip through a temporary device copy
  B2_CUDA(cudaMalloc(reinterpret_cast<void**>(&dev), bytes));
  int rc = B2_OK;
  if (cudaMemcpyAsync(dev, values, bytes, cudaMemcpyHostToDevice, ctx->stream) != cudaSuccess) rc = B2_E_CUDA;
  if (rc == B2_OK) rc = launch_softmax_rows(ctx, dev, n_rows, n_cols);
  if (rc == B2_OK && cudaMemcpyAsync(values, dev, bytes, cudaMemcpyDeviceToHost, ctx->stream) != cudaSuccess) rc = B2_E_CUDA;
  const cudaError_t done = cudaStreamSynchronize(ctx->stream);
  cudaFree(dev);
  if (rc == B2_E_CUDA) set_error("b2_softmax_rows: copying the host values failed");
  if (rc != B2_OK) return rc;
  B2_CUDA(done);
  return B2_OK;
}

// ---- LinearSVC / LinearSVR (DESIGN.md section 15) -------------------------------------------------------------------
// The operands go where the GLM passes keep theirs: the trial point as (w, b), the accepted point as (step, db), then
// 1 when there is an accepted point and the positive label (or eps) in the two label slots.
int b2_svm_pass(b2_ctx* ctx, const void* X, int x_dtype, const float* y, int64_t n_rows, int d, int64_t ldx,
                int mem_kind, const uint8_t* row_mask, int mask_keep, int loss, double pos_label_or_epsilon,
                const double* coef_from, double intercept_from, const double* coef, double intercept, int fit_intercept,
                double* sums_out, double* dhess_out) {
  if (int r = use_device(ctx)) return r;
  if (sums_out == nullptr) { set_error("sums_out is null"); return B2_E_ARG; }
  if (loss != B2_SVM_SQUARED_HINGE && loss != B2_SVM_SQUARED_EPSILON) {
    set_error("loss=%d must be B2_SVM_SQUARED_HINGE or B2_SVM_SQUARED_EPSILON", loss);
    return B2_E_ARG;
  }
  const double p = pos_label_or_epsilon;
  if (!isfinite(p) || (loss == B2_SVM_SQUARED_EPSILON && p < 0.0)) {
    set_error(loss == B2_SVM_SQUARED_HINGE ? "pos_label=%g must be finite" : "epsilon=%g must be finite and >= 0", p);
    return B2_E_ARG;
  }
  const std::vector<double> zero(kMaxD, 0.0);
  const bool has_from = coef_from != nullptr;
  if (int r = glm_operands(ctx, x_dtype, n_rows, d, ldx, mem_kind, X, y, true, coef, fit_intercept ? intercept : 0.0,
                           has_from ? coef_from : zero.data(), (has_from && fit_intercept) ? intercept_from : 0.0,
                           has_from ? 1.0 : 0.0, p))
    return r;
  const bool hess = dhess_out != nullptr;
  if (int r = row_pass(ctx, X, x_dtype, y, n_rows, d, ldx, mem_kind, row_mask, [&](const RowSpan& s, void*, void*, void*) {
        return launch_svm(ctx, s.X, x_dtype, s.rows, d, s.ldx, s.y, s.mask, mask_keep, loss, hess, s.first);
      }))
    return r;
  return fetch_glm_sums(ctx, d, 0, sums_out, dhess_out);
}

// ---- RidgeClassifierCV (DESIGN.md section 13) -----------------------------------------------------------------------
// Host rows with cv_out stream in blocks whose cv block stays within the 262 144 x 64 doubles of b2_ridge_loo's widest
constexpr size_t kLooOutBlockBytes = ((size_t)1 << 18) * kMaxAlphas * sizeof(double);

// The Gram of the kept rows, the class sums at its column means (b2_class_sums), the eigendecomposition of the centred
// Gram, one leave-one-out pass with T targets over the same rows, the first best alpha, then b2_solve_classes there.
int b2_ridge_classifier_loo(b2_ctx* ctx, const void* X, int x_dtype, const float* y, int64_t n_rows, int d, int64_t ldx,
                            int mem_kind, const uint8_t* row_mask, int mask_keep, const float* classes, int n_classes,
                            const double* alphas, int n_alphas, int fit_intercept, int scoring, double* mse_out,
                            double* correct_out, double* cv_out, int* best_out, double* coef_out, double* intercept_out,
                            double* counts_out) {
  if (int r = use_device(ctx)) return r;
  if (int r = check_shape(x_dtype, n_rows, d, ldx, mem_kind)) return r;
  if (alphas == nullptr || n_alphas < 1 || n_alphas > kMaxAlphas) {
    set_error("n_alphas=%d out of range [1,%d] (or alphas is null)", n_alphas, kMaxAlphas);
    return B2_E_ARG;
  }
  for (int a = 0; a < n_alphas; ++a)
    if (!(isfinite(alphas[a]) && alphas[a] > 0.0)) {
      set_error("alphas[%d] == %g, must be > 0.0 and finite", a, alphas[a]);
      return B2_E_ARG;
    }
  if (int r = check_classes(classes, n_classes)) return r;
  if (scoring != B2_LOO_SQUARED && scoring != B2_LOO_ACCURACY) {
    set_error("scoring=%d: B2_LOO_SQUARED or B2_LOO_ACCURACY expected", scoring);
    return B2_E_ARG;
  }
  if (mse_out == nullptr || correct_out == nullptr || best_out == nullptr || coef_out == nullptr ||
      intercept_out == nullptr || counts_out == nullptr) {
    set_error("mse_out / correct_out / best_out / coef_out / intercept_out / counts_out is null");
    return B2_E_ARG;
  }
  if (n_rows > 0 && (X == nullptr || y == nullptr)) { set_error("X / y is null"); return B2_E_ARG; }
  if (int r = ensure_cls(ctx, "b2_ridge_classifier_loo")) return r;
  if (ctx->loo_cls == nullptr) B2_CUDA(cudaMalloc(reinterpret_cast<void**>(&ctx->loo_cls), sizeof(double) * kLcDoubles));
  // (1) the Gram, (2) the class sums at its column means
  if (int r = b2_gram_reset(ctx, d)) return r;
  if (int r = gram_rows(ctx, X, x_dtype, y, n_rows, d, ldx, mem_kind, row_mask, mask_keep)) return r;
  std::vector<double> S((size_t)(d + 2) * (d + 2));
  if (int r = b2_gram_export(ctx, S.data(), nullptr)) return r;
  const double n_kept = S[(size_t)d * (d + 2) + d];
  if (!(n_kept > 0.0)) { set_error("no row kept: the leave-one-out error needs at least one row"); return B2_E_ARG; }
  std::vector<double> center(d), sums((size_t)n_classes * (d + 1));
  for (int j = 0; j < d; ++j) center[j] = S[(size_t)j * (d + 2) + d] / n_kept;
  if (int r = b2_class_sums(ctx, X, x_dtype, y, n_rows, d, ldx, mem_kind, row_mask, mask_keep, classes, n_classes,
                            fit_intercept ? center.data() : nullptr, sums.data(), counts_out))
    return r;
  // (3) the eigendecomposition, (4) the pass
  if (int r = launch_solve_eigh(ctx, fit_intercept)) return r;
  B2_CUDA(cudaMemcpyAsync(ctx->loo + kLooAlpha, alphas, sizeof(double) * n_alphas, cudaMemcpyHostToDevice, ctx->stream));
  double converged = 0.0;
  B2_CUDA(cudaMemcpyAsync(&converged, ctx->loo + kLooMisc + 3, sizeof(double), cudaMemcpyDeviceToHost, ctx->stream));
  B2_CUDA(cudaStreamSynchronize(ctx->stream));
  if (int r = eigh_converged(converged)) return r;
  const int T = n_classes == 2 ? 1 : n_classes;
  const size_t cv_row = sizeof(double) * T * n_alphas;
  const bool accuracy = scoring == B2_LOO_ACCURACY;
  if (int r = row_pass(
          ctx, X, x_dtype, y, n_rows, d, ldx, mem_kind, row_mask,
          [&](const RowSpan& s, void* cv, void*, void*) {
            return launch_loo_classes(ctx, s.X, x_dtype, s.rows, d, s.ldx, s.y, s.mask, mask_keep, n_classes, n_alphas,
                                      fit_intercept, accuracy, static_cast<double*>(cv), s.first);
          },
          RowOut{cv_out, cv_row}, {}, {}, cv_out != nullptr ? (int64_t)(kLooOutBlockBytes / cv_row) & ~(int64_t)31 : 0))
    return r;
  double h[kLcPart];
  B2_CUDA(cudaMemcpyAsync(h, ctx->loo_cls + kLcSum, sizeof(h), cudaMemcpyDeviceToHost, ctx->stream));
  B2_CUDA(cudaStreamSynchronize(ctx->stream));
  // (5) the first alpha with the strictly best score: the smallest mse, or the most rows right
  int best = 0;
  for (int a = 0; a < n_alphas; ++a) {
    mse_out[a] = h[a] / (n_kept * T);
    correct_out[a] = h[kMaxAlphas + a];
    const bool better = accuracy ? correct_out[a] > correct_out[best] : mse_out[a] < mse_out[best];
    if (better) best = a;
  }
  *best_out = best;
  // (6) the model there
  return b2_solve_classes(ctx, alphas[best], fit_intercept, nullptr, n_classes, coef_out, intercept_out);
}

// ---- scoring ---------------------------------------------------------------------------------------
int b2_score(b2_ctx* ctx, const void* X, int x_dtype, int64_t n_rows, int d, int64_t ldx, int mem_kind,
             const double* coef, double intercept, const float* y, const uint8_t* row_mask, int mask_keep,
             float* yhat, double* stats_out) {
  if (int r = use_device(ctx)) return r;
  if (int r = check_shape(x_dtype, n_rows, d, ldx, mem_kind)) return r;
  if (coef == nullptr || (n_rows > 0 && X == nullptr)) { set_error("coef / X is null"); return B2_E_ARG; }
  // coefficients go up through one of two pinned slots (no stream sync per call: the slot is only waited for when it
  // is reused, two calls later)
  {
    const int slot = ctx->coef_slot;
    ctx->coef_slot ^= 1;
    B2_CUDA(cudaEventSynchronize(ctx->ev_coef[slot]));
    double* cbuf = ctx->coef_host + (size_t)slot * (kMaxD + 1);
    memset(cbuf, 0, sizeof(double) * (kMaxD + 1));
    memcpy(cbuf, coef, sizeof(double) * d);
    cbuf[kMaxD] = intercept;
    B2_CUDA(cudaMemcpyAsync(ctx->coef_dev, cbuf, sizeof(double) * (kMaxD + 1), cudaMemcpyHostToDevice, ctx->stream));
    B2_CUDA(cudaEventRecord(ctx->ev_coef[slot], ctx->stream));
  }
  double* acc = score_totals(ctx);
  if (n_rows == 0) {
    B2_CUDA(cudaMemsetAsync(acc, 0, sizeof(double) * kNStats, ctx->stream));
  } else if (int r = row_pass(
                 ctx, X, x_dtype, y, n_rows, d, ldx, mem_kind, row_mask,
                 [&](const RowSpan& s, void* yh, void*, void*) {
                   return launch_score(ctx, s.X, x_dtype, s.rows, d, s.ldx, s.y, s.mask, mask_keep,
                                       static_cast<float*>(yh), s.first);
                 },
                 RowOut{yhat, sizeof(float)})) {
    return r;
  }
  if (stats_out != nullptr && y != nullptr) {
    B2_CUDA(cudaMemcpyAsync(stats_out, acc, sizeof(double) * kNStats, cudaMemcpyDeviceToHost, ctx->stream));
    B2_CUDA(cudaStreamSynchronize(ctx->stream));
  }
  return B2_OK;
}

int b2_score_allreduce(b2_ctx* ctx, double* stats) {
  if (int r = use_device(ctx)) return r;
  if (stats == nullptr) { set_error("stats is null"); return B2_E_ARG; }
  if (ctx->comm == nullptr) {
    if (ctx->n_ranks > 1) { set_error("b2_score_allreduce needs the NCCL communicator (b2_comm_init)"); return B2_E_STATE; }
    return B2_OK;
  }
  NcclApi* api = nccl();
  if (api == nullptr) { set_error("libnccl.so.2 could not be loaded"); return B2_E_COMM; }
  double* acc = score_totals(ctx);   // kNStats sums
  double* mx = acc + kNStats;         // 2 maxima
  B2_CUDA(cudaStreamSynchronize(ctx->stream));   // the previous b2_score may still be reading its totals
  double host[kNStats], hmax[2];
  memcpy(host, stats, sizeof(host));
  hmax[0] = host[4]; hmax[1] = host[9];
  host[4] = 0.0; host[9] = 0.0;
  B2_CUDA(cudaMemcpyAsync(acc, host, sizeof(host), cudaMemcpyHostToDevice, ctx->stream));
  B2_CUDA(cudaMemcpyAsync(mx, hmax, sizeof(hmax), cudaMemcpyHostToDevice, ctx->stream));
  B2_CUDA(cudaStreamSynchronize(ctx->stream));   // host / hmax live on this stack frame
  B2_NCCL(api, api->AllReduce(acc, acc, kNStats, kNcclFloat64, kNcclSum, ctx->comm, ctx->stream));
  B2_NCCL(api, api->AllReduce(mx, mx, 2, kNcclFloat64, kNcclMax, ctx->comm, ctx->stream));
  B2_CUDA(cudaMemcpyAsync(host, acc, sizeof(host), cudaMemcpyDeviceToHost, ctx->stream));
  B2_CUDA(cudaMemcpyAsync(hmax, mx, sizeof(hmax), cudaMemcpyDeviceToHost, ctx->stream));
  B2_CUDA(cudaStreamSynchronize(ctx->stream));
  host[4] = hmax[0]; host[9] = hmax[1];
  memcpy(stats, host, sizeof(host));
  return B2_OK;
}

// ---- synthetic rows -------------------------------------------------------------------------------------
int b2_synth(b2_ctx* ctx, uint64_t seed, int64_t row_offset, int64_t n_rows, int d, int64_t ldx, int x_dtype,
             double alpha, double beta, double sigma, void* X_dev, float* y_dev) {
  if (int r = use_device(ctx)) return r;
  if (int r = check_shape(x_dtype, n_rows, d, ldx, B2_MEM_DEVICE)) return r;
  if (n_rows > 0 && (X_dev == nullptr || y_dev == nullptr)) { set_error("X / y is null"); return B2_E_ARG; }
  return launch_synth(ctx, seed, row_offset, n_rows, d, ldx, x_dtype, alpha, beta, sigma, X_dev, y_dev);
}

// y >= 0 filtered one-feature tranche of day `day` (stage_3_synthetic_data_generation.py:28-43)
int b2_synth_tranche(b2_ctx* ctx, uint64_t seed, int64_t n_rows, int day, double beta, double sigma, float* X_dev,
                     float* y_dev, int64_t* n_kept_out) {
  if (int r = use_device(ctx)) return r;
  if (n_rows < 0 || day < 1 || n_kept_out == nullptr || (n_rows > 0 && (X_dev == nullptr || y_dev == nullptr))) {
    set_error("bad arguments to b2_synth_tranche");
    return B2_E_ARG;
  }
  if (ctx->synth_count == nullptr) B2_CUDA(cudaMalloc(reinterpret_cast<void**>(&ctx->synth_count), 16));
  // alpha(d) = kappa + amplitude * sin(2 pi f (d - 1) / 364), kappa = 1, amplitude = 0.5, f = 6  (stage_3...:31-33,38)
  const double alpha = 1.0 + 0.5 * sin(2.0 * 3.14159265358979323846 * 6.0 * (double)(day - 1) / 364.0);
  if (int r = launch_synth_tranche(ctx, seed, n_rows, alpha, beta, sigma, X_dev, y_dev,
                                   reinterpret_cast<int64_t*>(ctx->synth_count)))
    return r;
  long long kept = 0;
  B2_CUDA(cudaMemcpyAsync(&kept, ctx->synth_count, sizeof(kept), cudaMemcpyDeviceToHost, ctx->stream));
  B2_CUDA(cudaStreamSynchronize(ctx->stream));
  *n_kept_out = (int64_t)kept;
  return B2_OK;
}

// ---- model_metrics on two vectors (stage_1_train_model.py:79-90), fp32 or fp64 inputs -------------------------
int b2_metrics(b2_ctx* ctx, const void* y_actual, const void* y_predicted, int dtype, int64_t n_rows, int mem_kind,
               double* stats_out) {
  if (int r = use_device(ctx)) return r;
  if (dtype != B2_F32 && dtype != B2_F64) { set_error("dtype must be B2_F32 or B2_F64"); return B2_E_ARG; }
  if (n_rows < 0 || stats_out == nullptr || (n_rows > 0 && (y_actual == nullptr || y_predicted == nullptr))) {
    set_error("bad arguments to b2_metrics");
    return B2_E_ARG;
  }
  if (mem_kind != B2_MEM_DEVICE && mem_kind != B2_MEM_HOST) { set_error("bad mem_kind %d", mem_kind); return B2_E_ARG; }
  double* acc = score_totals(ctx);
  const size_t es = dtype == B2_F32 ? 4 : 8;
  if (n_rows == 0) {
    B2_CUDA(cudaMemsetAsync(acc, 0, sizeof(double) * kNStats, ctx->stream));
  } else if (mem_kind == B2_MEM_DEVICE) {
    if (int r = launch_metrics(ctx, y_actual, y_predicted, dtype, n_rows, true)) return r;
  } else {
    // host vectors: blocks through the two staging buffers of the streamed paths (x block = y_actual, y block region
    // is too small for fp64, so both vectors share the X block: [rows] actual then [rows] predicted)
    if (int r = ensure_staging(ctx)) return r;
    const int64_t blk_rows = (int64_t)(ctx->stage_bytes_x / (2 * es));
    if (int r = stream_host_blocks(
            ctx, n_rows, blk_rows,
            [&](int buf, int64_t r0, int64_t rows) -> int {
              char* dst = static_cast<char*>(ctx->stage_x[buf]);
              const size_t off = (size_t)r0 * es, bytes = (size_t)rows * es;
              B2_CUDA(cudaMemcpyAsync(dst, static_cast<const char*>(y_actual) + off, bytes, cudaMemcpyHostToDevice,
                                      ctx->copy_stream));
              B2_CUDA(cudaMemcpyAsync(dst + (size_t)blk_rows * es, static_cast<const char*>(y_predicted) + off, bytes,
                                      cudaMemcpyHostToDevice, ctx->copy_stream));
              return B2_OK;
            },
            [&](int buf, int64_t r0, int64_t rows) {
              const char* src = static_cast<const char*>(ctx->stage_x[buf]);
              return launch_metrics(ctx, src, src + (size_t)blk_rows * es, dtype, rows, r0 == 0);
            }))
      return r;
  }
  B2_CUDA(cudaMemcpyAsync(stats_out, acc, sizeof(double) * kNStats, cudaMemcpyDeviceToHost, ctx->stream));
  B2_CUDA(cudaStreamSynchronize(ctx->stream));
  return B2_OK;
}

// counters of the context: [0] b2_fit calls whose device rows ended on the tensor-core kernel, [1] exchanges started,
// [2] kernels launched
int b2_ctx_stats(b2_ctx* ctx, int64_t* out3) {
  if (ctx == nullptr || out3 == nullptr) { set_error("null argument"); return B2_E_ARG; }
  out3[0] = ctx->fused_fits;
  out3[1] = (int64_t)ctx->xchg_epoch;
  out3[2] = ctx->launches;
  return B2_OK;
}

// ---- multi-GPU --------------------------------------------------------------------------------------------
int b2_comm_unique_id(char* id_out) {
  if (id_out == nullptr) { set_error("id_out is null"); return B2_E_ARG; }
  NcclApi* api = nccl();
  if (api == nullptr) { set_error("libnccl.so.2 could not be loaded"); return B2_E_COMM; }
  NcclUid uid;
  B2_NCCL(api, api->GetUniqueId(&uid));
  memcpy(id_out, uid.internal, 128);
  return B2_OK;
}

int b2_comm_init(b2_ctx* ctx, int n_ranks, int rank, const char* id) {
  if (int r = use_device(ctx)) return r;
  if (n_ranks < 1 || rank < 0 || rank >= n_ranks || id == nullptr) { set_error("bad communicator arguments"); return B2_E_ARG; }
  if (ctx->comm != nullptr) { set_error("communicator already initialised"); return B2_E_STATE; }
  NcclApi* api = nccl();
  if (api == nullptr) { set_error("libnccl.so.2 could not be loaded"); return B2_E_COMM; }
  NcclUid uid;
  memcpy(uid.internal, id, 128);
  B2_NCCL(api, api->CommInitRank(&ctx->comm, n_ranks, uid, rank));
  ctx->n_ranks = n_ranks;
  ctx->rank = rank;
  return B2_OK;
}

int b2_comm_destroy(b2_ctx* ctx) {
  if (ctx == nullptr || ctx->comm == nullptr) return B2_OK;
  NcclApi* api = nccl();
  if (api != nullptr && api->CommDestroy != nullptr) api->CommDestroy(ctx->comm);
  ctx->comm = nullptr;
  ctx->n_ranks = 1;
  ctx->rank = 0;
  return B2_OK;
}

static int ensure_xchg(b2_ctx* ctx) {
  if (ctx->xchg == nullptr) {
    B2_CUDA(cudaMalloc(reinterpret_cast<void**>(&ctx->xchg), kXchgBytes));
    B2_CUDA(cudaMemset(ctx->xchg, 0, kXchgBytes));
    B2_CUDA(cudaDeviceSynchronize());
  }
  return B2_OK;
}

int b2_comm_p2p_export(b2_ctx* ctx, char* handle_out) {
  if (int r = use_device(ctx)) return r;
  if (handle_out == nullptr) { set_error("handle_out is null"); return B2_E_ARG; }
  if (int r = ensure_xchg(ctx)) return r;
  cudaIpcMemHandle_t h;
  B2_CUDA(cudaIpcGetMemHandle(&h, ctx->xchg));
  static_assert(sizeof(h) == 64, "cudaIpcMemHandle_t is 64 bytes");
  memcpy(handle_out, &h, 64);
  return B2_OK;
}

// A (re-)attached exchange starts at exchange number 0 on every rank: clear this rank's flags, ticket and status
// (stale numbers from an earlier attachment would satisfy the first wait at once).  The caller's rendezvous must put
// a barrier between the attach of all ranks and the first exchange -- peers write into this buffer.
static int reset_exchange_words(b2_ctx* ctx) {
  B2_CUDA(cudaStreamSynchronize(ctx->stream));
  B2_CUDA(cudaMemset(xchg_flags(ctx->xchg), 0, 256));
  B2_CUDA(cudaDeviceSynchronize());
  ctx->xchg_epoch = 0;
  ctx->xchg_pending = false;
  ctx->xchg_status_host[0] = 0u;
  return B2_OK;
}

int b2_comm_p2p_attach(b2_ctx* ctx, int n_ranks, int rank, const char* handles) {
  if (int r = use_device(ctx)) return r;
  if (n_ranks < 2 || n_ranks > kMaxRanks || rank < 0 || rank >= n_ranks || handles == nullptr || ctx->xchg == nullptr) {
    set_error("b2_comm_p2p_attach: bad arguments (2..%d ranks; call b2_comm_p2p_export first)", kMaxRanks);
    return B2_E_ARG;
  }
  if (ctx->p2p_ready) { set_error("peer exchange already attached"); return B2_E_STATE; }
  if (int r = reset_exchange_words(ctx)) return r;
  for (int r = 0; r < n_ranks; ++r) {
    if (r == rank) { ctx->xchg_peer[r] = ctx->xchg; continue; }
    cudaIpcMemHandle_t h;
    memcpy(&h, handles + (size_t)r * 64, 64);
    void* p = nullptr;
    B2_CUDA(cudaIpcOpenMemHandle(&p, h, cudaIpcMemLazyEnablePeerAccess));
    ctx->xchg_peer[r] = static_cast<double*>(p);
  }
  ctx->n_ranks = n_ranks;
  ctx->rank = rank;
  ctx->p2p_ready = true;
  ctx->p2p_local = false;
  return B2_OK;
}

// Same exchange between contexts of ONE process (a C client driving several GPUs, or two contexts on one GPU): the
// peers' buffers are ordinary device pointers, reached through cudaDeviceEnablePeerAccess when the devices differ.
int b2_comm_p2p_attach_local(b2_ctx* ctx, int n_ranks, int rank, b2_ctx* const* peers) {
  if (int r = use_device(ctx)) return r;
  if (n_ranks < 2 || n_ranks > kMaxRanks || rank < 0 || rank >= n_ranks || peers == nullptr || peers[rank] != ctx) {
    set_error("b2_comm_p2p_attach_local: bad arguments (2..%d contexts, peers[rank] == ctx)", kMaxRanks);
    return B2_E_ARG;
  }
  if (ctx->p2p_ready) { set_error("peer exchange already attached"); return B2_E_STATE; }
  for (int r = 0; r < n_ranks; ++r) {
    if (peers[r] == nullptr) { set_error("peers[%d] is null", r); return B2_E_ARG; }
    B2_CUDA(cudaSetDevice(peers[r]->device));
    if (int rc = ensure_xchg(peers[r])) return rc;
  }
  B2_CUDA(cudaSetDevice(ctx->device));
  if (int r = reset_exchange_words(ctx)) return r;
  for (int r = 0; r < n_ranks; ++r) {
    if (peers[r]->device != ctx->device) {
      int can = 0;
      B2_CUDA(cudaDeviceCanAccessPeer(&can, ctx->device, peers[r]->device));
      if (!can) { set_error("device %d cannot map the memory of device %d", ctx->device, peers[r]->device); return B2_E_UNSUPPORTED; }
      const cudaError_t e = cudaDeviceEnablePeerAccess(peers[r]->device, 0);
      if (e != cudaSuccess && e != cudaErrorPeerAccessAlreadyEnabled) B2_CUDA(e);
      cudaGetLastError();
    }
    ctx->xchg_peer[r] = peers[r]->xchg;
  }
  // contexts that share ONE device: a peer's kernel waiting for this rank's flags holds an SM, and the cooperative Gram
  // launch needs all of its CTAs resident at once -- leave those SMs free (a test / single-GPU configuration)
  int same_device = 0;
  for (int r = 0; r < n_ranks; ++r) same_device += (r != rank && peers[r]->device == ctx->device) ? 1 : 0;
  if (same_device > 0 && ctx->sm_limit == 0) { ctx->sm_limit = ctx->sm_count - 9 * same_device; ctx->sm_limit_auto = true; }
  ctx->n_ranks = n_ranks;
  ctx->rank = rank;
  ctx->p2p_ready = true;
  ctx->p2p_local = true;
  return B2_OK;
}

int b2_comm_p2p_detach(b2_ctx* ctx) {
  if (ctx == nullptr) { set_error("null context"); return B2_E_ARG; }
  cudaSetDevice(ctx->device);
  cudaStreamSynchronize(ctx->stream);
  if (ctx->p2p_ready && !ctx->p2p_local)
    for (int r = 0; r < ctx->n_ranks; ++r)
      if (r != ctx->rank && ctx->xchg_peer[r] != nullptr) cudaIpcCloseMemHandle(ctx->xchg_peer[r]);
  for (int r = 0; r < kMaxRanks; ++r) ctx->xchg_peer[r] = nullptr;
  if (ctx->p2p_ready && ctx->comm == nullptr) { ctx->n_ranks = 1; ctx->rank = 0; }
  if (ctx->sm_limit_auto) { ctx->sm_limit = 0; ctx->sm_limit_auto = false; }
  ctx->p2p_ready = false;
  ctx->p2p_local = false;
  cudaGetLastError();
  return B2_OK;
}

int b2_comm_set_timeout_ms(b2_ctx* ctx, int64_t ms) {
  if (ctx == nullptr || ms < 1) { set_error("timeout must be >= 1 ms"); return B2_E_ARG; }
  ctx->xchg_timeout_ns = (unsigned long long)ms * 1000000ull;
  return B2_OK;
}

int b2_comm_info(b2_ctx* ctx, int* n_ranks_out, int* rank_out, int* exchange_out) {
  if (ctx == nullptr) { set_error("null context"); return B2_E_ARG; }
  if (n_ranks_out != nullptr) *n_ranks_out = ctx->n_ranks;
  if (rank_out != nullptr) *rank_out = ctx->rank;
  if (exchange_out != nullptr)
    *exchange_out = (ctx->n_ranks > 1 && ctx->p2p_ready) ? B2_EXCHANGE_PEER : (ctx->comm != nullptr ? B2_EXCHANGE_NCCL : B2_EXCHANGE_NONE);
  return B2_OK;
}

int b2_comm_barrier(b2_ctx* ctx) {
  if (int r = use_device(ctx)) return r;
  if (ctx->comm == nullptr) return b2_ctx_sync(ctx);
  NcclApi* api = nccl();
  if (api == nullptr) { set_error("libnccl.so.2 could not be loaded"); return B2_E_COMM; }
  double* slot = ctx->tc_red + kTcAccElems + 8;  // spare scratch
  B2_NCCL(api, api->AllReduce(slot, slot, 1, kNcclFloat64, kNcclSum, ctx->comm, ctx->stream));
  B2_CUDA(cudaStreamSynchronize(ctx->stream));
  return B2_OK;
}

// ---- timing ---------------------------------------------------------------------------------------------------
int b2_timer_start(b2_ctx* ctx) {
  if (int r = use_device(ctx)) return r;
  B2_CUDA(cudaEventRecord(ctx->ev_t0, ctx->stream));
  return B2_OK;
}
int b2_timer_stop(b2_ctx* ctx, double* ms_out) {
  if (int r = use_device(ctx)) return r;
  B2_CUDA(cudaEventRecord(ctx->ev_t1, ctx->stream));
  B2_CUDA(cudaEventSynchronize(ctx->ev_t1));
  float ms = 0.f;
  B2_CUDA(cudaEventElapsedTime(&ms, ctx->ev_t0, ctx->ev_t1));
  if (ms_out != nullptr) *ms_out = (double)ms;
  return B2_OK;
}
int b2_last_kernel_ms(b2_ctx* ctx, double* gram_ms_out, int* launches_out) {
  if (int r = use_device(ctx)) return r;
  double total = 0.0;
  const int n = ctx->k_pairs < kKernelEventPairs ? ctx->k_pairs : kKernelEventPairs;
  for (int i = 0; i < n; ++i) {
    B2_CUDA(cudaEventSynchronize(ctx->ev_k[i][1]));
    float ms = 0.f;
    B2_CUDA(cudaEventElapsedTime(&ms, ctx->ev_k[i][0], ctx->ev_k[i][1]));
    total += ms;
  }
  if (gram_ms_out != nullptr) *gram_ms_out = total;
  if (launches_out != nullptr) *launches_out = n;
  ctx->k_pairs = 0;
  return B2_OK;
}
int b2_launch_count(b2_ctx* ctx, int64_t* n_out) {
  if (ctx == nullptr || n_out == nullptr) { set_error("null argument"); return B2_E_ARG; }
  *n_out = ctx->launches;
  return B2_OK;
}

}  // extern "C"
