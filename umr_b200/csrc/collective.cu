// collective.cu -- the ONE exchange of the data-parallel render step (SURVEY.md §8e): all-reduce of the flat
// shared-parameter gradient [V*3 + F*T2*3] (0.56 MB at C2), as our own one-shot kernel over NVLink peer memory.
//
// Reference equivalent: the implicit gradient reduce of torch.nn.DataParallel (experiments/train_s2.py:101,133,149,164).
//
// The raster backward accumulates the gradient into a SYMMETRIC buffer (same allocation on every rank, mapped into
// every peer's address space).  One kernel per rank then
//   1. tells every peer "my buffer is complete" (release store to the peer's flag word, system scope) and waits for
//      all peers' flags (acquire loads) -- block 0, then released to the other blocks through a device-scope flag;
//   2. sums the N buffers with 128-bit loads straight from peer memory (N * 0.56 MB over NVLink per GPU, every rank
//      computes the full sum itself: one-shot, latency-optimal at this size) and writes average/sum to a local output;
//   3. the last block to finish tells every peer "I am done reading you" and waits for the same from all of them, so
//      the next step may overwrite the symmetric buffer when this kernel has completed.
// It is a plain kernel: it is captured in the step's CUDA graph with everything else (the round-1 step kept an eager
// ncclAllReduce + mul + 4 pack/unpack copies outside the graph).  NCCL remains the fallback (umr_b200/dist.py).
#include <cuda_runtime.h>
#include <stdint.h>

#include "common.cuh"
#include "umr_b200.h"

namespace umr {

__device__ __forceinline__ void st_release_sys(uint32_t* p, uint32_t v) {
    asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ uint32_t ld_acquire_sys(const uint32_t* p) {
    uint32_t v;
    asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ void st_release_gpu(uint32_t* p, uint32_t v) {
    asm volatile("st.release.gpu.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ uint32_t ld_acquire_gpu(const uint32_t* p) {
    uint32_t v;
    asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}
// peer memory must not be served from this SM's L1 (it may hold last step's lines)
__device__ __forceinline__ float4 ld_peer_f4(const float4* p) {
    float4 v;
    asm volatile("ld.volatile.global.v4.f32 {%0,%1,%2,%3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "l"(p) : "memory");
    return v;
}

constexpr int AR_MAX_WORLD = 16;
// flag words at the end of every rank's symmetric buffer (uint32, zero-initialised once):
//   [0, 16)  arrive[r]: written by rank r        [16, 32) done[r]: written by rank r
// local (non-symmetric, zero-initialised) state `loc`: [0] ready flag (block 0 -> other blocks), [1] last completed
// epoch, [2] finished-block counter

__global__ void __launch_bounds__(256) k_p2p_allreduce(const uint64_t* __restrict__ peer_bufs, float* __restrict__ out,
                                                       size_t n4, size_t flag_off_bytes, uint32_t* __restrict__ loc,
                                                       int rank, int world, float scale) {
    __shared__ uint32_t s_epoch;
    const int tid = threadIdx.x;
    // this launch's epoch: 1 + the epoch of the previous launch, which its LAST block stored in loc[1] before exiting
    // (stable for the whole of this launch: it is only rewritten at the very end, after every block has passed its wait)
    if (tid == 0) s_epoch = loc[1] + 1u;
    __syncthreads();
    const uint32_t epoch = s_epoch;
    // ---- 1. cross-rank "inputs complete" ------------------------------------------------------------------
    if (blockIdx.x == 0) {
        if (tid < world) {
            __threadfence_system();  // the gradient written by earlier kernels on this GPU is visible to the peers
            uint32_t* peer_flags = reinterpret_cast<uint32_t*>(peer_bufs[tid] + flag_off_bytes);
            st_release_sys(peer_flags + rank, epoch);
            const uint32_t* mine = reinterpret_cast<const uint32_t*>(peer_bufs[rank] + flag_off_bytes);
            while ((int32_t)(ld_acquire_sys(mine + tid) - epoch) < 0) {}
        }
        __syncthreads();
        if (tid == 0) st_release_gpu(loc + 0, epoch);  // release the other blocks of this GPU
    } else {
        if (tid == 0) {
            while ((int32_t)(ld_acquire_gpu(loc + 0) - epoch) < 0) {}
        }
        __syncthreads();
    }
    // ---- 2. sum the peers' buffers ---------------------------------------------------------------------------
    for (size_t i = (size_t)blockIdx.x * blockDim.x + tid; i < n4; i += (size_t)gridDim.x * blockDim.x) {
        float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
        // all peer loads of a batch are issued before the first one is consumed (one NVLink round trip per batch of 8
        // ranks instead of one per rank); summed in rank order on every rank: bit-identical results everywhere
        for (int r0 = 0; r0 < world; r0 += 8) {
            float4 v[8];
#pragma unroll
            for (int q = 0; q < 8; ++q)
                if (r0 + q < world) v[q] = ld_peer_f4(reinterpret_cast<const float4*>(peer_bufs[r0 + q]) + i);
#pragma unroll
            for (int q = 0; q < 8; ++q)
                if (r0 + q < world) { acc.x += v[q].x; acc.y += v[q].y; acc.z += v[q].z; acc.w += v[q].w; }
        }
        reinterpret_cast<float4*>(out)[i] = make_float4(acc.x * scale, acc.y * scale, acc.z * scale, acc.w * scale);
    }
    // ---- 3. cross-rank "done reading" (last block) ---------------------------------------------------------------
    __syncthreads();
    __shared__ bool s_last;
    if (tid == 0) {
        __threadfence();
        s_last = atomicAdd(loc + 2, 1u) == gridDim.x - 1;
    }
    __syncthreads();
    if (s_last) {
        if (tid < world) {
            uint32_t* peer_flags = reinterpret_cast<uint32_t*>(peer_bufs[tid] + flag_off_bytes);
            st_release_sys(peer_flags + AR_MAX_WORLD + rank, epoch);
            const uint32_t* mine = reinterpret_cast<const uint32_t*>(peer_bufs[rank] + flag_off_bytes);
            while ((int32_t)(ld_acquire_sys(mine + AR_MAX_WORLD + tid) - epoch) < 0) {}
        }
        __syncthreads();
        if (tid == 0) {
            loc[2] = 0u;     // block counter for the next launch
            loc[1] = epoch;  // last completed epoch
        }
    }
}

}  // namespace umr

using namespace umr;

extern "C" size_t umr_p2p_allreduce_flag_bytes(void) { return 2 * AR_MAX_WORLD * sizeof(uint32_t); }

extern "C" int umr_p2p_allreduce(const void* peer_buffers_dev, float* out, int64_t n_floats, int64_t flag_offset_bytes,
                                 void* local_state, int32_t rank, int32_t world, float scale, void* stream_) {
    if (!peer_buffers_dev || !out || !local_state || n_floats <= 0 || (n_floats & 3) != 0) return UMR_ERR_BAD_ARG;
    if (world < 1 || world > AR_MAX_WORLD || rank < 0 || rank >= world) return UMR_ERR_BAD_ARG;
    if ((flag_offset_bytes & 15) != 0 || flag_offset_bytes < n_floats * 4) return UMR_ERR_BAD_ARG;
    cudaStream_t st = (cudaStream_t)stream_;
    const size_t n4 = (size_t)n_floats / 4;
    // every block must be resident at once (blocks wait for block 0): at most one block per SM
    int dev = 0, sms = 0;
    cudaError_t e = cudaGetDevice(&dev);
    if (e != cudaSuccess) return (int)e;
    e = cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    if (e != cudaSuccess) return (int)e;
    unsigned grid = (unsigned)((n4 + 255) / 256);
    if (grid > (unsigned)sms) grid = (unsigned)sms;
    if (grid < 1) grid = 1;
    launch(k_p2p_allreduce, grid, 256, 0, st, (const uint64_t*)peer_buffers_dev, out, n4, (size_t)flag_offset_bytes,
           (uint32_t*)local_state, rank, world, scale);
    return (int)cudaGetLastError();
}
