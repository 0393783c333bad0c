// c_api.cu -- error strings / version for the C ABI (include/umr_b200.h).
#include <cuda_runtime.h>

#include "umr_b200.h"

extern "C" const char* umr_error_string(int code) {
    switch (code) {
        case UMR_OK: return "ok";
        case UMR_ERR_UNSUPPORTED: return "mode not supported by the sm_90a kernels";
        case UMR_ERR_BAD_ARG: return "bad argument (null pointer, non-positive size or misaligned buffer)";
        case UMR_ERR_TOO_LARGE: return "size exceeds a compiled limit";
        default: break;
    }
    if (code > 0) return cudaGetErrorString((cudaError_t)code);
    return "unknown error";
}

extern "C" int umr_version(void) { return 204; }  // 200: round-2 ABI (pair buffer, workspace size takes the image size); 201: color_channels, texture-only backward; 202: umr_nmr_*; 203: 32-byte pair records; 204: umr_voxelize*
extern "C" size_t umr_sizeof_raster_params(void) { return sizeof(UmrRasterParams); }
extern "C" size_t umr_sizeof_project_params(void) { return sizeof(UmrProjectParams); }

#include <atomic>
namespace umr { std::atomic<unsigned long long> g_launches{0}; }
extern "C" uint64_t umr_launch_count(void) { return umr::g_launches.load(); }
extern "C" int umr_event_create(void** event) {
    if (!event) return UMR_ERR_BAD_ARG;
    cudaEvent_t e;
    cudaError_t rc = cudaEventCreate(&e);
    *event = (void*)e;
    return (int)rc;
}
extern "C" int umr_event_destroy(void* event) { return (int)cudaEventDestroy((cudaEvent_t)event); }
extern "C" int umr_event_record(void* event, void* stream) {
    return (int)cudaEventRecord((cudaEvent_t)event, (cudaStream_t)stream);
}
extern "C" int umr_event_elapsed_ms(void* start, void* stop, float* ms) {
    if (!ms) return UMR_ERR_BAD_ARG;
    cudaError_t rc = cudaEventSynchronize((cudaEvent_t)stop);
    if (rc != cudaSuccess) return (int)rc;
    return (int)cudaEventElapsedTime(ms, (cudaEvent_t)start, (cudaEvent_t)stop);
}
