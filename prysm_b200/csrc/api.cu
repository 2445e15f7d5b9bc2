// Handle lifetime, scratch arenas, tensor-map encoding, error reporting.
#include "common.cuh"

namespace pb {

int ensure_scratch(Handle* h, int slot, size_t bytes, void** out) {
    if (bytes > h->scratch_bytes[slot]) {
        if (h->scratch[slot]) {
            // an earlier call may still be reading the old arena on some stream
            PB_CUDA(h, cudaDeviceSynchronize());
            PB_CUDA(h, cudaFree(h->scratch[slot]));
            h->scratch[slot] = nullptr;
            h->scratch_bytes[slot] = 0;
        }
        size_t want = bytes + bytes / 8;
        if (cudaMalloc(&h->scratch[slot], want) != cudaSuccess) {
            cudaGetLastError();
            return fail(h, PB_ERR_ALLOC, "scratch allocation of " + std::to_string(want) + " bytes failed");
        }
        h->scratch_bytes[slot] = want;
    }
    *out = h->scratch[slot];
    return PB_OK;
}

int fold_scratch(Handle* h, int rows, int blocks, int per, cudaStream_t st, double** part, unsigned** counters) {
    void* w = nullptr;
    const size_t bytes = (size_t)rows * blocks * per * sizeof(double);
    PB_TRY(ensure_scratch(h, FOLD_SLOT, bytes + (size_t)rows * sizeof(unsigned), &w));
    *part = (double*)w;
    *counters = (unsigned*)((char*)w + bytes);
    PB_CUDA(h, cudaMemsetAsync(*counters, 0, (size_t)rows * sizeof(unsigned), st));
    return PB_OK;
}

int encode_tensor_map(Handle* h, CUtensorMap* map, CUtensorMapDataType type, int rank, const void* base,
                      const cuuint64_t* dims, const cuuint64_t* strides_bytes, const cuuint32_t* box,
                      CUtensorMapSwizzle swizzle, CUtensorMapL2promotion l2) {
    typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                      const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                      CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
    static EncodeTiledFn fn = nullptr;   // a driver entry point: process-wide, not per device
    if (!fn) {
        cudaDriverEntryPointQueryResult q;
        void* f = nullptr;
        PB_CUDA(h, cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &f, cudaEnableDefault, &q));
        if (!f || q != cudaDriverEntryPointSuccess) return fail(h, PB_ERR_CUDA, "cuTensorMapEncodeTiled not available");
        fn = reinterpret_cast<EncodeTiledFn>(f);
    }
    const cuuint32_t estr[5] = {1, 1, 1, 1, 1};
    CUresult r = fn(map, type, (cuuint32_t)rank, const_cast<void*>(base), dims, strides_bytes, box, estr,
                    CU_TENSOR_MAP_INTERLEAVE_NONE, swizzle, l2, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) return fail(h, PB_ERR_CUDA, "cuTensorMapEncodeTiled failed with CUresult " + std::to_string((int)r));
    return PB_OK;
}

}  // namespace pb

using namespace pb;

extern "C" int pb_create(pb_handle_t* out, int device) {
    if (!out) return PB_ERR_INVALID;
    *out = nullptr;
    int count = 0;
    if (cudaGetDeviceCount(&count) != cudaSuccess || device < 0 || device >= count) return PB_ERR_CUDA;
    DeviceGuard guard(device);   // the caller's current device is restored on return
    int cur = -1;
    if (cudaGetDevice(&cur) != cudaSuccess || cur != device) return PB_ERR_CUDA;
    if (cudaFree(0) != cudaSuccess) return PB_ERR_CUDA;   // make sure the device's primary context exists
    Handle* h = new Handle();
    h->device = device;
    cudaDeviceGetAttribute(&h->sm_count, cudaDevAttrMultiProcessorCount, device);
    cudaDeviceGetAttribute(&h->max_smem_optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, device);
    *out = reinterpret_cast<pb_handle_t>(h);
    return PB_OK;
}

extern "C" int pb_destroy(pb_handle_t hh) {
    Handle* h = reinterpret_cast<Handle*>(hh);
    if (!h) return PB_OK;
    DeviceGuard guard(h->device);
    cudaDeviceSynchronize();
    for (auto& kv : h->tables) cudaFree(kv.second);
    for (void* p : h->scratch) if (p) cudaFree(p);
    for (auto& e : h->side_ev) if (e) cudaEventDestroy(e);
    if (h->side) cudaStreamDestroy(h->side);
    delete h;
    return PB_OK;
}

extern "C" const char* pb_last_error(pb_handle_t hh) {
    Handle* h = reinterpret_cast<Handle*>(hh);
    return h ? h->err.c_str() : "null handle";
}

extern "C" const char* pb_version(void) { return "prysm_b200 0.1 (sm_90a)"; }

extern "C" long long pb_launch_count(pb_handle_t hh) {
    Handle* h = reinterpret_cast<Handle*>(hh);
    return h ? h->launches : 0;
}

extern "C" long long pb_route_launch_count(pb_handle_t hh, int route) {
    Handle* h = reinterpret_cast<Handle*>(hh);
    if (!h) return PB_ERR_INVALID;
    auto it = h->route_launches.find(route);
    return it == h->route_launches.end() ? 0 : it->second;
}
