// Context, scratch arenas and error reporting of libalq.
#include <initializer_list>
#include <mutex>
#include <new>

#include "alq_common.cuh"

extern "C" int alq_version(void) { return 10; }

extern "C" int alq_create(alq_ctx** out, int device) {
    if (!out) return ALQ_ERR_INVALID;
    *out = nullptr;
    int count = 0;
    if (cudaGetDeviceCount(&count) != cudaSuccess || device < 0 || device >= count) {
        cudaGetLastError();
        return ALQ_ERR_CUDA;  // no CPU fallback: without a usable GPU there is no context
    }
    alq_ctx* ctx = new (std::nothrow) alq_ctx();
    if (!ctx) return ALQ_ERR_NOMEM;
    ctx->device = device;
    cudaDeviceProp prop;
    if (cudaSetDevice(device) != cudaSuccess || cudaGetDeviceProperties(&prop, device) != cudaSuccess) {
        delete ctx;
        return ALQ_ERR_CUDA;
    }
    if (prop.major != 9 || prop.minor != 0) {
        delete ctx;
        return ALQ_ERR_CUDA;  // built for sm_90a only
    }
    ctx->sm_count = prop.multiProcessorCount;
    if (prop.clockRate > 0) ctx->clock_khz = prop.clockRate;
    ctx->smem_optin = prop.sharedMemPerBlockOptin;
    cudaStreamCreateWithFlags(&ctx->side_stream, cudaStreamNonBlocking);
    cudaStreamCreateWithFlags(&ctx->side_stream2, cudaStreamNonBlocking);
    cudaEventCreate(&ctx->ev_a);
    cudaEventCreate(&ctx->ev_b);
    if (cudaHostAlloc(reinterpret_cast<void**>(&ctx->xchg_status_host), sizeof(int), cudaHostAllocMapped) == cudaSuccess) {
        *ctx->xchg_status_host = 0;
        cudaHostGetDevicePointer(reinterpret_cast<void**>(&ctx->xchg_status_dev), ctx->xchg_status_host, 0);
    } else {
        cudaGetLastError();
    }
    *out = ctx;
    return ALQ_OK;
}

extern "C" void alq_destroy(alq_ctx* ctx) {
    if (!ctx) return;
    cudaSetDevice(ctx->device);
    alq_comm_destroy(ctx);
    if (ctx->scratch) cudaFree(ctx->scratch);
    if (ctx->arena2) cudaFree(ctx->arena2);
    if (ctx->tile_counters) cudaFree(ctx->tile_counters);
    if (ctx->sel_ring) cudaFree(ctx->sel_ring);
    if (ctx->pinned) cudaFreeHost(ctx->pinned);
    if (ctx->xchg_status_host) cudaFreeHost(ctx->xchg_status_host);
    if (ctx->side_stream) cudaStreamDestroy(ctx->side_stream);
    if (ctx->side_stream2) cudaStreamDestroy(ctx->side_stream2);
    if (ctx->ev_a) cudaEventDestroy(ctx->ev_a);
    if (ctx->ev_b) cudaEventDestroy(ctx->ev_b);
    delete ctx;
}

namespace {
// Kernels with device-wide spin barriers (the fused tail, the persistent selection loop) need all of their CTAs resident,
// so two of them must never share the device.  Launches on ONE stream are ordered anyway; only when the stream changes
// is the previous stream fenced with an event (recorded then, lazily: it also covers whatever was enqueued behind the
// last such kernel, which only over-synchronises).  begin() .. end() hold the lock across the launch.
std::mutex g_gridsync_mu;
cudaEvent_t g_gridsync_ev[64] = {};
cudaStream_t g_gridsync_last[64] = {};
bool g_gridsync_has[64] = {};
}  // namespace

void alq_gridsync_begin(alq_ctx* ctx, cudaStream_t st) {
    g_gridsync_mu.lock();
    const int d = ctx->device & 63;
    if (!g_gridsync_has[d] || g_gridsync_last[d] == st) return;
    if (!g_gridsync_ev[d]) cudaEventCreateWithFlags(&g_gridsync_ev[d], cudaEventDisableTiming);
    if (g_gridsync_ev[d] && cudaEventRecord(g_gridsync_ev[d], g_gridsync_last[d]) == cudaSuccess) cudaStreamWaitEvent(st, g_gridsync_ev[d], 0);
    else cudaGetLastError();            // the previous stream no longer exists: its work is already draining
}

void alq_gridsync_end(alq_ctx* ctx, cudaStream_t st) {
    const int d = ctx->device & 63;
    g_gridsync_last[d] = st;
    g_gridsync_has[d] = true;
    g_gridsync_mu.unlock();
}

extern "C" const char* alq_last_error(const alq_ctx* ctx) {
    return ctx ? ctx->err.c_str() : "null context";
}

extern "C" int alq_set_option(alq_ctx* ctx, const char* key, int64_t value) {
    if (!ctx || !key) return ALQ_ERR_INVALID;
    const std::string k(key);
    if (k == "k3_impl" && value >= 0 && value <= 2) ctx->k3_impl = static_cast<int>(value);
    else if (k == "greedy_variant" && value >= 0 && value <= 3) ctx->greedy_variant = static_cast<int>(value);
    else if (k == "l2_resident_mb" && value >= 0 && value <= 4096) ctx->l2_resident_mb = static_cast<int>(value);
    else if (k == "d2_fast_path" && value >= 0 && value <= 1) ctx->d2_fast_path = static_cast<int>(value);
    else if (k == "tail_buckets" && value >= 0 && value <= 1) ctx->tail_buckets = static_cast<int>(value);
    else if (k == "spin_timeout_ms" && value >= 1 && value <= 3600000) ctx->spin_timeout_ms = static_cast<int>(value);
    else if (k == "select_impl" && value >= 0 && value <= 2) ctx->select_impl = static_cast<int>(value);
    else if (k == "base_impl" && value >= 0 && value <= 2) ctx->base_impl = static_cast<int>(value);
    else if (k == "balancing_loop" && value >= 0 && value <= 3) ctx->balancing_loop = static_cast<int>(value);
    else ALQ_FAIL(ctx, ALQ_ERR_INVALID, "alq_set_option: unknown option or value: %s=%lld", key, (long long)value);
    return ALQ_OK;
}

extern "C" int64_t alq_launch_count(const alq_ctx* ctx) { return ctx ? ctx->launches : 0; }

int alq_scratch_reserve(alq_ctx* ctx, size_t bytes) {
    if (bytes <= ctx->scratch_bytes) return ALQ_OK;
    // grow-only; callers never hold scratch pointers across API calls
    ALQ_CUDA(ctx, cudaDeviceSynchronize());
    if (ctx->scratch) cudaFree(ctx->scratch);
    ctx->scratch = nullptr;
    ctx->scratch_bytes = 0;
    size_t want = bytes + (bytes >> 2) + (1u << 20);
    if (cudaMalloc(&ctx->scratch, want) != cudaSuccess) {
        cudaGetLastError();
        ALQ_FAIL(ctx, ALQ_ERR_NOMEM, "scratch allocation of %zu bytes failed", want);
    }
    ctx->scratch_bytes = want;
    return ALQ_OK;
}

int alq_pinned_reserve(alq_ctx* ctx, size_t bytes) {
    if (bytes <= ctx->pinned_bytes) return ALQ_OK;
    if (ctx->pinned) cudaFreeHost(ctx->pinned);
    if (ctx->xchg_status_host) cudaFreeHost(ctx->xchg_status_host);
    ctx->pinned = nullptr;
    ctx->pinned_bytes = 0;
    if (cudaMallocHost(&ctx->pinned, bytes) != cudaSuccess) {
        cudaGetLastError();
        ALQ_FAIL(ctx, ALQ_ERR_NOMEM, "pinned allocation of %zu bytes failed", bytes);
    }
    ctx->pinned_bytes = bytes;
    return ALQ_OK;
}

int alq_arena2_reserve(alq_ctx* ctx, size_t bytes) {
    if (bytes <= ctx->arena2_bytes) return ALQ_OK;
    ALQ_CUDA(ctx, cudaDeviceSynchronize());
    if (ctx->arena2) cudaFree(ctx->arena2);
    ctx->arena2 = nullptr;
    ctx->arena2_bytes = 0;
    if (cudaMalloc(&ctx->arena2, bytes) != cudaSuccess) {
        cudaGetLastError();
        ALQ_FAIL(ctx, ALQ_ERR_NOMEM, "arena2 allocation of %zu bytes failed", bytes);
    }
    ctx->arena2_bytes = bytes;
    return ALQ_OK;
}
