// Runtime plumbing of libadaqp_b200: error reporting, device slabs, CUDA IPC.
// Replaces the pinned-host buffer registry of AdaQP/communicator/buffer.py:154-248
// with device-resident, peer-mapped slabs (see include/adaqp_b200.h).
#include <stdarg.h>
#include <string.h>

#include "common.cuh"

static thread_local char g_err[512] = "";

void adaqp_set_error(const char *fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
}

int adaqp_check_launch(const char *what) {
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) {
        adaqp_set_error("%s launch failed: %s", what, cudaGetErrorString(e));
        return (int)e;
    }
    return 0;
}

AdaqpOptions &adaqp_options() {
    static AdaqpOptions opt = {1, 0, 8, 0, 0, 0, 32, 0};
    return opt;
}

namespace {
int *option_slot(const char *name) {
    AdaqpOptions &o = adaqp_options();
    if (!name) return nullptr;
    if (!strcmp(name, "spmm_impl")) return &o.spmm_impl;
    if (!strcmp(name, "spmm_rows_per_grab")) return &o.spmm_rows_per_grab;
    if (!strcmp(name, "spmm_ctas_per_sm")) return &o.spmm_ctas_per_sm;
    if (!strcmp(name, "spmm_hints")) return &o.spmm_hints;
    if (!strcmp(name, "exch_send_ctas")) return &o.exch_send_ctas;
    if (!strcmp(name, "exch_recv_ctas")) return &o.exch_recv_ctas;
    if (!strcmp(name, "gemm_block_k")) return &o.gemm_block_k;
    if (!strcmp(name, "spmm_slice_cols")) return &o.spmm_slice_cols;
    return nullptr;
}
}  // namespace

extern "C" {

int adaqp_abi_version(void) { return ADAQP_ABI_VERSION; }

int adaqp_set_option(const char *name, int64_t value) {
    int *slot = option_slot(name);
    ADAQP_REQUIRE(slot != nullptr, ADAQP_EINVAL, "adaqp_set_option: unknown option '%s'", name ? name : "(null)");
    ADAQP_REQUIRE(value >= 0 && value <= (1 << 20), ADAQP_EINVAL, "adaqp_set_option: %s=%lld out of range", name, (long long)value);
    *slot = (int)value;
    return 0;
}

int adaqp_get_option(const char *name, int64_t *value) {
    int *slot = option_slot(name);
    ADAQP_REQUIRE(slot != nullptr && value != nullptr, ADAQP_EINVAL, "adaqp_get_option: unknown option '%s'", name ? name : "(null)");
    *value = *slot;
    return 0;
}

int adaqp_enable_peer_access(int peer_device) {
    int dev = 0;
    ADAQP_CUDA(cudaGetDevice(&dev));
    if (dev == peer_device) return 0;
    int can = 0;
    ADAQP_CUDA(cudaDeviceCanAccessPeer(&can, dev, peer_device));
    ADAQP_REQUIRE(can, ADAQP_EINVAL, "adaqp_enable_peer_access: device %d cannot map device %d", dev, peer_device);
    const cudaError_t e = cudaDeviceEnablePeerAccess(peer_device, 0);
    if (e == cudaErrorPeerAccessAlreadyEnabled) { (void)cudaGetLastError(); return 0; }
    ADAQP_CUDA(e);
    return 0;
}

const char *adaqp_last_error(void) { return g_err; }

int adaqp_sm_count(void) {
    int dev = 0, n = 0;
    if (cudaGetDevice(&dev) != cudaSuccess) return -1;
    if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess) return -1;
    return n;
}

int adaqp_slab_alloc(void **ptr, size_t bytes) {
    ADAQP_REQUIRE(ptr != nullptr && bytes > 0, ADAQP_EINVAL, "adaqp_slab_alloc: bad arguments");
    ADAQP_CUDA(cudaMalloc(ptr, bytes));
    ADAQP_CUDA(cudaMemset(*ptr, 0, bytes));
    ADAQP_CUDA(cudaDeviceSynchronize());
    return 0;
}

int adaqp_slab_free(void *ptr) {
    if (ptr) ADAQP_CUDA(cudaFree(ptr));
    return 0;
}

int adaqp_ipc_export(void *ptr, unsigned char handle[ADAQP_IPC_HANDLE_BYTES]) {
    static_assert(sizeof(cudaIpcMemHandle_t) == ADAQP_IPC_HANDLE_BYTES, "IPC handle size");
    ADAQP_REQUIRE(ptr && handle, ADAQP_EINVAL, "adaqp_ipc_export: null argument");
    cudaIpcMemHandle_t h;
    ADAQP_CUDA(cudaIpcGetMemHandle(&h, ptr));
    memcpy(handle, &h, sizeof(h));
    return 0;
}

int adaqp_ipc_open(const unsigned char handle[ADAQP_IPC_HANDLE_BYTES], void **ptr) {
    ADAQP_REQUIRE(ptr && handle, ADAQP_EINVAL, "adaqp_ipc_open: null argument");
    cudaIpcMemHandle_t h;
    memcpy(&h, handle, sizeof(h));
    ADAQP_CUDA(cudaIpcOpenMemHandle(ptr, h, cudaIpcMemLazyEnablePeerAccess));
    return 0;
}

int adaqp_ipc_close(void *ptr) {
    if (ptr) ADAQP_CUDA(cudaIpcCloseMemHandle(ptr));
    return 0;
}

int adaqp_can_access_peer(int peer_device) {
    int dev = 0, can = 0;
    if (cudaGetDevice(&dev) != cudaSuccess) return 0;
    if (dev == peer_device) return 1;
    if (cudaDeviceCanAccessPeer(&can, dev, peer_device) != cudaSuccess) return 0;
    return can;
}

}  // extern "C"
