// Peer-memory windows for the multi-GPU selection loop (one process per GPU on one NVSwitch node).
// Every rank cudaMalloc's one window, exports it with cudaIpcGetMemHandle; the 64-byte handles are
// exchanged by the caller (torch.distributed all_gather: plumbing), and every rank maps its peers'
// windows with cudaIpcOpenMemHandle.  After that the kernels in alq_greedy.cu exchange per-step
// winners / running min-distances with plain st.global / ld.global on those mapped pointers (NVLink
// P2P) and system-scope flags -- no host round trip and no collective library inside the 10 000-step loop.
#include "alq_common.cuh"

namespace {

struct PeerWindows {
    char* p[ALQ_MAX_WORLD];
};

__global__ void comm_ready_kernel(const __grid_constant__ PeerWindows W, int world, int rank, unsigned long long tag) {
    if (threadIdx.x < world) {
        __threadfence_system();
        st_release_sys(reinterpret_cast<unsigned long long*>(W.p[threadIdx.x]) + rank, tag);
    }
}

}  // namespace

int alq_comm_ready(alq_ctx* ctx, unsigned long long tag, cudaStream_t st) {
    PeerWindows W{};
    for (int r = 0; r < ctx->comm.world; ++r) W.p[r] = ctx->comm.peer[r];
    comm_ready_kernel<<<1, 32, 0, st>>>(W, ctx->comm.world, ctx->comm.rank, tag);
    ALQ_LAUNCH_CHECK(ctx);
    return ALQ_OK;
}

extern "C" int alq_comm_create(alq_ctx* ctx, int32_t world, int32_t rank, size_t window_bytes, void* handle_out) {
    if (!ctx) return ALQ_ERR_INVALID;
    if (world < 1 || world > ALQ_MAX_WORLD || rank < 0 || rank >= world || !handle_out || window_bytes < (1u << 16))
        ALQ_FAIL(ctx, ALQ_ERR_INVALID, "alq_comm_create: bad arguments (world=%d rank=%d, max world %d)", world, rank, ALQ_MAX_WORLD);
    if (ctx->comm.window) ALQ_FAIL(ctx, ALQ_ERR_STATE, "alq_comm_create: a group already exists on this context");
    ALQ_CUDA(ctx, cudaSetDevice(ctx->device));
    void* w = nullptr;
    if (cudaMalloc(&w, window_bytes) != cudaSuccess) {
        cudaGetLastError();
        ALQ_FAIL(ctx, ALQ_ERR_NOMEM, "alq_comm_create: window allocation of %zu bytes failed", window_bytes);
    }
    ALQ_CUDA(ctx, cudaMemset(w, 0, window_bytes));
    cudaIpcMemHandle_t h;
    if (cudaIpcGetMemHandle(&h, w) != cudaSuccess) {
        const char* e = cudaGetErrorString(cudaGetLastError());
        cudaFree(w);
        ALQ_FAIL(ctx, ALQ_ERR_CUDA, "cudaIpcGetMemHandle failed: %s", e);
    }
    static_assert(sizeof(cudaIpcMemHandle_t) == ALQ_IPC_HANDLE_BYTES, "IPC handle size");
    memcpy(handle_out, &h, sizeof(h));
    ctx->comm.world = world;
    ctx->comm.rank = rank;
    ctx->comm.window = static_cast<char*>(w);
    ctx->comm.bytes = window_bytes;
    ctx->comm.epoch = 0;
    for (int i = 0; i < ALQ_MAX_WORLD; ++i) ctx->comm.peer[i] = nullptr;
    ctx->comm.peer[rank] = ctx->comm.window;
    ctx->comm.connected = (world == 1);
    return ALQ_OK;
}

extern "C" int alq_comm_connect(alq_ctx* ctx, const void* all_handles) {
    if (!ctx || !all_handles) return ALQ_ERR_INVALID;
    if (!ctx->comm.window) ALQ_FAIL(ctx, ALQ_ERR_STATE, "alq_comm_connect: call alq_comm_create first");
    ALQ_CUDA(ctx, cudaSetDevice(ctx->device));
    const char* hs = static_cast<const char*>(all_handles);
    for (int r = 0; r < ctx->comm.world; ++r) {
        if (r == ctx->comm.rank || ctx->comm.peer[r]) continue;
        cudaIpcMemHandle_t h;
        memcpy(&h, hs + static_cast<size_t>(r) * ALQ_IPC_HANDLE_BYTES, sizeof(h));
        void* p = nullptr;
        cudaError_t e = cudaIpcOpenMemHandle(&p, h, cudaIpcMemLazyEnablePeerAccess);
        if (e != cudaSuccess) {
            cudaGetLastError();
            ALQ_FAIL(ctx, ALQ_ERR_CUDA, "cudaIpcOpenMemHandle(rank %d) failed: %s (needs NVLink/PCIe peer access)", r,
                     cudaGetErrorString(e));
        }
        ctx->comm.peer[r] = static_cast<char*>(p);
    }
    ctx->comm.connected = true;
    return ALQ_OK;
}

extern "C" int alq_comm_destroy(alq_ctx* ctx) {
    if (!ctx) return ALQ_ERR_INVALID;
    if (!ctx->comm.window) return ALQ_OK;
    cudaSetDevice(ctx->device);
    cudaDeviceSynchronize();
    for (int r = 0; r < ctx->comm.world; ++r)
        if (r != ctx->comm.rank && ctx->comm.peer[r]) cudaIpcCloseMemHandle(ctx->comm.peer[r]);
    cudaFree(ctx->comm.window);
    ctx->comm = AlqComm{};
    return ALQ_OK;
}

// Exportable device memory for one rank's band of Ward's condensed distances (alq_ward_nn_chain_banded): a cudaMalloc
// allocation of its own, since an IPC handle names the base of an allocation (a sub-allocated block of a caching
// allocator cannot be exported on its own).
extern "C" int alq_band_alloc(alq_ctx* ctx, size_t bytes, void** ptr_out, void* handle_out) {
    if (!ctx) return ALQ_ERR_INVALID;
    if (!bytes || !ptr_out || !handle_out) ALQ_FAIL(ctx, ALQ_ERR_INVALID, "alq_band_alloc: bad arguments (bytes=%zu)", bytes);
    ALQ_CUDA(ctx, cudaSetDevice(ctx->device));
    void* p = nullptr;
    if (cudaMalloc(&p, bytes) != cudaSuccess) {
        cudaGetLastError();
        ALQ_FAIL(ctx, ALQ_ERR_NOMEM, "alq_band_alloc: allocation of %zu bytes failed", bytes);
    }
    cudaIpcMemHandle_t h;
    if (cudaIpcGetMemHandle(&h, p) != cudaSuccess) {
        const char* e = cudaGetErrorString(cudaGetLastError());
        cudaFree(p);
        ALQ_FAIL(ctx, ALQ_ERR_CUDA, "alq_band_alloc: cudaIpcGetMemHandle failed: %s", e);
    }
    memcpy(handle_out, &h, sizeof(h));
    *ptr_out = p;
    return ALQ_OK;
}

extern "C" int alq_band_open(alq_ctx* ctx, const void* handle, void** ptr_out) {
    if (!ctx) return ALQ_ERR_INVALID;
    if (!handle || !ptr_out) ALQ_FAIL(ctx, ALQ_ERR_INVALID, "alq_band_open: bad arguments");
    ALQ_CUDA(ctx, cudaSetDevice(ctx->device));
    cudaIpcMemHandle_t h;
    memcpy(&h, handle, sizeof(h));
    void* p = nullptr;
    const cudaError_t e = cudaIpcOpenMemHandle(&p, h, cudaIpcMemLazyEnablePeerAccess);
    if (e != cudaSuccess) {
        cudaGetLastError();
        ALQ_FAIL(ctx, ALQ_ERR_CUDA, "alq_band_open: cudaIpcOpenMemHandle failed: %s (needs NVLink/PCIe peer access)",
                 cudaGetErrorString(e));
    }
    *ptr_out = p;
    return ALQ_OK;
}

extern "C" int alq_band_close(alq_ctx* ctx, void* ptr) {
    if (!ctx) return ALQ_ERR_INVALID;
    if (!ptr) ALQ_FAIL(ctx, ALQ_ERR_INVALID, "alq_band_close: null pointer");
    ALQ_CUDA(ctx, cudaSetDevice(ctx->device));
    ALQ_CUDA(ctx, cudaIpcCloseMemHandle(ptr));
    return ALQ_OK;
}

extern "C" int alq_band_free(alq_ctx* ctx, void* ptr) {
    if (!ctx) return ALQ_ERR_INVALID;
    if (!ptr) ALQ_FAIL(ctx, ALQ_ERR_INVALID, "alq_band_free: null pointer");
    ALQ_CUDA(ctx, cudaSetDevice(ctx->device));
    ALQ_CUDA(ctx, cudaFree(ptr));
    return ALQ_OK;
}
