// Gradient all-reduce over NVLink peer memory — the library's own exchange: no NCCL and no host on the
// data path, every piece an ordinary node of the step's CUDA graph.
//
// Replaces the Horovod call of the reference's data-parallel path
// (utils/distributed.py:16-43: flatten -> hvd.allreduce_ (mean) -> unflatten; call sites
// train_vqa.py:193-199, pretrain.py:302-308).  Every rank holds the same flat gradient arena
// (uniter_b200/arena.py); the arenas, one staging buffer and one 256-byte signal block per rank
// are mapped into every process with cudaIpc (NVSwitch: every peer at full bandwidth).
//
// Protocol (two-shot; the slice [offset, offset+count) is cut into `world` sub-slices of `per`
// 16-byte vectors):
//   A  push   : rank r copies its sub-slice q (q != r) into stage_q[r]
//      barrier 1: signal PUSH[r] = epoch on every peer, wait for PUSH[q] >= epoch from all q
//   C  reduce : rank r sums its own sub-slice r and the world-1 staged copies in fp32 (fixed rank
//               order -> every rank ends up with bit-identical values), scales (1/world = the
//               mean Horovod computes) and the result goes into sub-slice r of EVERY arena
//      barrier 2: signal BCAST[r] = epoch on every peer, wait for BCAST[q] >= epoch from all q
// Epochs are monotonic and live in device memory, so replaying the same captured nodes is correct.
// Hazards: a rank can only enter call e+1 after every peer signalled BCAST of call e, i.e. after
// every peer has finished reading its staging buffer and this rank's arena.  Spin waits are bounded
// (~20 s): on expiry a sticky error word is set and every later wait of this rank returns at once
// (wrong data, but never a hung GPU); the host checks the word.
//
// Three forms of the same protocol (ub200_peer_allreduce_args.max_ctas), in the order they were built;
//
//   > 0  peer_allreduce_kernel: ONE persistent kernel, both phases with SM loads / posted remote stores.
//        256 threads x <= 64 registers, no shared memory, so a CTA fits next to a persistent GEMM CTA
//        (384 x <= 168 registers) — but 16 K registers hold only ~32 KB in flight, so it needs most
//        of the SMs to approach NVLink bandwidth.
//   = 0  peer_push_kernel + peer_reduce_kernel: work-sized grids of short-lived CTAs.
//   < 0  (default) the COPY ENGINES move the bytes (cudaMemcpyAsync nodes), peer_sync_kernel runs the
//        barriers, peer_reduce_local_kernel reduces out of local HBM: nothing competes with the
//        backward pass the exchange overlaps — the only form that gained from the overlap.
#include <cudaTypedefs.h>
#include <string.h>

#include "common.h"
#include "ptx.cuh"

namespace ub {

constexpr int PEER_MAX = UB200_MAX_PEERS;
// signal block layout (uint32 words)
constexpr int PF_PUSH = 0;      // [8]  written by peer q: pushes of call `epoch` have landed here
constexpr int PF_BCAST = 8;     // [8]  written by peer q: its reduced sub-slice has landed here
constexpr int PF_EPOCH = 16;    // local: number of completed calls
constexpr int PF_ARRIVE_A = 17; // local: CTAs that finished phase A
constexpr int PF_ARRIVE_C = 18; // local: CTAs that finished phase C
constexpr int PF_ERROR = 19;    // local, sticky: (epoch << 4) | phase of the first expired wait
constexpr int PF_WORDS = 64;

struct PeerParams {
  uint8_t* buf[PEER_MAX];
  uint8_t* stage[PEER_MAX];
  uint32_t* flags[PEER_MAX];
  int rank, world;
  long long byte_offset;   // of the slice inside the arena
  long long nvec;          // 16-byte vectors in the slice
  long long per;           // vectors per sub-slice (multiple of 32)
  float scale;
  long long timeout_cycles;
};

__device__ __forceinline__ void st_release_sys(uint32_t* p, uint32_t v) {
  asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ uint32_t ld_acquire_sys(const uint32_t* p) {
  uint32_t v;
  asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ uint32_t ld_relaxed_sys(const uint32_t* p) {
  uint32_t v;
  asm volatile("ld.relaxed.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}

// wait until *flag >= epoch (wrap-safe); false if the wait expired or an error is already latched
__device__ __forceinline__ bool peer_wait(uint32_t* mine, int word, uint32_t epoch, int phase,
                                          long long timeout) {
  if (ld_relaxed_sys(mine + PF_ERROR) != 0) return false;
  const long long t0 = clock64();
  int spins = 0;
  while (static_cast<int32_t>(ld_acquire_sys(mine + word) - epoch) < 0) {
    if ((++spins & 1023) == 0) {
      if (clock64() - t0 > timeout || ld_relaxed_sys(mine + PF_ERROR) != 0) {
        atomicCAS(mine + PF_ERROR, 0u, (epoch << 4) | static_cast<uint32_t>(phase));
        return false;
      }
    }
    __nanosleep(64);
  }
  return true;
}

template <bool kBF16>
__device__ __forceinline__ void acc8(float (&a)[8], const uint4& v) {
  float2 f;
  f = Elem<kBF16>::unpack(v.x); a[0] += f.x; a[1] += f.y;
  f = Elem<kBF16>::unpack(v.y); a[2] += f.x; a[3] += f.y;
  f = Elem<kBF16>::unpack(v.z); a[4] += f.x; a[5] += f.y;
  f = Elem<kBF16>::unpack(v.w); a[6] += f.x; a[7] += f.y;
}

template <bool kBF16>
__global__ void __launch_bounds__(256, 4) peer_allreduce_kernel(const PeerParams p) {
  uint32_t* mine = p.flags[p.rank];
  const int tid = threadIdx.x, lane = tid & 31;
  const int warp_g = blockIdx.x * (blockDim.x >> 5) + (tid >> 5);
  const int nwarps = gridDim.x * (blockDim.x >> 5);
  // every CTA reads the same value: the word is bumped by the LAST CTA of a call, after all have arrived
  const uint32_t epoch = ld_relaxed_sys(mine + PF_EPOCH) + 1u;
  const long long chunks = p.per >> 5;   // 32-vector (512-byte) warp chunks per sub-slice

  // ------------------------------------------------------------ A: push my copy of sub-slice q to rank q
  {
    const uint4* src0 = reinterpret_cast<const uint4*>(p.buf[p.rank] + p.byte_offset);
    // 32-bit index arithmetic: a slice has < 2^31 vectors (ub200_peer_allreduce checks)
    const uint32_t wm1 = static_cast<uint32_t>(p.world - 1);
    const uint32_t units = static_cast<uint32_t>(chunks) * wm1;
    const uint32_t per = static_cast<uint32_t>(p.per), nvec = static_cast<uint32_t>(p.nvec);
    for (uint32_t u0 = warp_g; u0 < units; u0 += 4u * nwarps) {
      uint4 v[4];
      uint32_t dsti[4];
      int q[4];
      bool on[4];
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const uint32_t u = u0 + static_cast<uint32_t>(k) * nwarps;
        on[k] = false;
        if (u < units && u >= u0) {
          const uint32_t c = u / wm1;
          const uint32_t j = u - c * wm1;
          q[k] = static_cast<int>((p.rank + 1 + j) % p.world);
          const uint32_t vi = c * 32 + lane;                // vector inside the sub-slice
          const uint32_t gi = q[k] * per + vi;              // vector inside the slice
          if (gi < nvec) {
            v[k] = src0[gi];
            dsti[k] = p.rank * per + vi;
            on[k] = true;
          }
        }
      }
#pragma unroll
      for (int k = 0; k < 4; ++k)
        if (on[k]) reinterpret_cast<uint4*>(p.stage[q[k]])[dsti[k]] = v[k];
    }
  }
  __syncthreads();
  if (tid == 0) {
    __threadfence_system();
    if (atomicAdd(mine + PF_ARRIVE_A, 1u) == gridDim.x - 1) {   // last CTA of this rank: all pushes issued
      mine[PF_ARRIVE_A] = 0;
      __threadfence_system();
      for (int q = 0; q < p.world; ++q) st_release_sys(p.flags[q] + PF_PUSH + p.rank, epoch);
    }
  }
  if (tid < p.world) peer_wait(mine, PF_PUSH + tid, epoch, 1, p.timeout_cycles);
  __syncthreads();

  // ------------------------------------------------------------ C: reduce sub-slice `rank`, write it everywhere
  {
    const long long v_lo = p.rank * p.per;
    const long long v_hi = min(p.nvec, v_lo + p.per);
    const uint4* own = reinterpret_cast<const uint4*>(p.buf[p.rank] + p.byte_offset);
    const uint4* stg = reinterpret_cast<const uint4*>(p.stage[p.rank]);
    for (long long c0 = warp_g; c0 * 32 < v_hi - v_lo; c0 += 2ll * nwarps) {
      float a[2][8];
      long long vi[2];
#pragma unroll
      for (int k = 0; k < 2; ++k) {
        vi[k] = (c0 + static_cast<long long>(k) * nwarps) * 32 + lane;
#pragma unroll
        for (int i = 0; i < 8; ++i) a[k][i] = 0.f;
      }
      for (int r = 0; r < p.world; ++r) {          // fixed order 0..world-1
        uint4 v[2];
#pragma unroll
        for (int k = 0; k < 2; ++k) {
          v[k] = make_uint4(0, 0, 0, 0);
          if (v_lo + vi[k] < v_hi) v[k] = (r == p.rank) ? own[v_lo + vi[k]] : stg[r * p.per + vi[k]];
        }
#pragma unroll
        for (int k = 0; k < 2; ++k) acc8<kBF16>(a[k], v[k]);
      }
#pragma unroll
      for (int k = 0; k < 2; ++k) {
        if (v_lo + vi[k] >= v_hi) continue;
        uint4 o;
        o.x = Elem<kBF16>::pack(a[k][0] * p.scale, a[k][1] * p.scale);
        o.y = Elem<kBF16>::pack(a[k][2] * p.scale, a[k][3] * p.scale);
        o.z = Elem<kBF16>::pack(a[k][4] * p.scale, a[k][5] * p.scale);
        o.w = Elem<kBF16>::pack(a[k][6] * p.scale, a[k][7] * p.scale);
        for (int j = 0; j < p.world; ++j) {
          const int q = (p.rank + j) % p.world;
          reinterpret_cast<uint4*>(p.buf[q] + p.byte_offset)[v_lo + vi[k]] = o;
        }
      }
    }
  }
  __syncthreads();
  if (tid == 0) {
    __threadfence_system();
    if (atomicAdd(mine + PF_ARRIVE_C, 1u) == gridDim.x - 1) {   // last CTA: everything of this rank is out
      mine[PF_ARRIVE_C] = 0;
      __threadfence_system();
      for (int q = 0; q < p.world; ++q) st_release_sys(p.flags[q] + PF_BCAST + p.rank, epoch);
      for (int q = 0; q < p.world; ++q) peer_wait(mine, PF_BCAST + q, epoch, 2, p.timeout_cycles);
      mine[PF_EPOCH] = epoch;
      __threadfence_system();
    }
  }
}

// ------------------------------------------------------------------------------------------------
// Form 2 (max_ctas == 0): the same protocol as TWO kernels of many short-lived CTAs.
// A persistent exchange CTA holds 16 K registers of its SM for the whole exchange: while it is there,
// the register-hungry row kernels of the backward (LayerNorm backward: 61 K registers per CTA,
// attention backward: 2 x 32 K) cannot be placed on that SM, and the chain the exchange is supposed to
// hide behind slows down.  Here every CTA moves 32 KB (push) / 8 KB (reduce) and exits, the grids are
// sized by the work, and the stream they run on has a LOWER priority than the backward's stream:
// the block scheduler places the backward's CTAs first and the exchange fills what is left — next to
// the persistent GEMM CTAs (80-96 registers x 512 threads leave room for exactly one 16 K-register CTA).
//   peer_push_kernel    grid (per / 2048, world - 1): block (x, y) copies vectors [2048 x, 2048 (x + 1)) of
//                       sub-slice q = rank + 1 + y into stage_q[rank]; destinations rotate with the rank so
//                       that no rank's ingress sees all senders at once.  Last CTA: PUSH signals.
//   peer_reduce_kernel  grid (per / 512): waits for every PUSH signal, reduces 512 vectors of sub-slice
//                       `rank`, writes them into every arena.  Last CTA: BCAST signals, waits for the
//                       peers' BCAST signals, bumps the epoch.
constexpr int PUSH_U = 8, PUSH_VPC = 256 * PUSH_U;      // vectors per push CTA
constexpr int RED_U = 2, RED_VPC = 256 * RED_U;          // vectors per reduce CTA

__global__ void __launch_bounds__(256, 4) peer_push_kernel(const PeerParams p) {
  uint32_t* mine = p.flags[p.rank];
  const uint32_t epoch = ld_relaxed_sys(mine + PF_EPOCH) + 1u;
  const int q = (p.rank + 1 + static_cast<int>(blockIdx.y)) % p.world;
  const uint32_t per = static_cast<uint32_t>(p.per), nvec = static_cast<uint32_t>(p.nvec);
  const uint32_t v0 = blockIdx.x * PUSH_VPC + threadIdx.x;
  const uint4* src = reinterpret_cast<const uint4*>(p.buf[p.rank] + p.byte_offset) + static_cast<size_t>(q) * per;
  uint4* dst = reinterpret_cast<uint4*>(p.stage[q]) + static_cast<size_t>(p.rank) * per;
  const uint32_t q_len = (static_cast<uint32_t>(q) * per < nvec) ? min(per, nvec - q * per) : 0u;
  uint4 v[PUSH_U];
#pragma unroll
  for (int k = 0; k < PUSH_U; ++k) {
    const uint32_t vi = v0 + k * 256;
    if (vi < q_len) v[k] = src[vi];
  }
#pragma unroll
  for (int k = 0; k < PUSH_U; ++k) {
    const uint32_t vi = v0 + k * 256;
    if (vi < q_len) dst[vi] = v[k];
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    __threadfence_system();
    const uint32_t total = gridDim.x * gridDim.y;
    if (atomicAdd(mine + PF_ARRIVE_A, 1u) == total - 1) {
      mine[PF_ARRIVE_A] = 0;
      __threadfence_system();
      for (int r = 0; r < p.world; ++r) st_release_sys(p.flags[r] + PF_PUSH + p.rank, epoch);
    }
  }
}

template <bool kBF16>
__global__ void __launch_bounds__(256, 4) peer_reduce_kernel(const PeerParams p) {
  uint32_t* mine = p.flags[p.rank];
  const int tid = threadIdx.x;
  const uint32_t epoch = ld_relaxed_sys(mine + PF_EPOCH) + 1u;
  // (this rank's own pushes are complete by stream order: the push kernel precedes this one)
  if (tid < p.world && tid != p.rank) peer_wait(mine, PF_PUSH + tid, epoch, 1, p.timeout_cycles);
  __syncthreads();
  const uint32_t per = static_cast<uint32_t>(p.per), nvec = static_cast<uint32_t>(p.nvec);
  const uint32_t v_lo = static_cast<uint32_t>(p.rank) * per;
  const uint32_t len = (v_lo < nvec) ? min(per, nvec - v_lo) : 0u;
  const uint4* own = reinterpret_cast<const uint4*>(p.buf[p.rank] + p.byte_offset) + v_lo;
  const uint4* stg = reinterpret_cast<const uint4*>(p.stage[p.rank]);
  float a[RED_U][8];
  uint32_t vi[RED_U];
#pragma unroll
  for (int k = 0; k < RED_U; ++k) {
    vi[k] = blockIdx.x * RED_VPC + k * 256 + tid;
#pragma unroll
    for (int i = 0; i < 8; ++i) a[k][i] = 0.f;
  }
  for (int r = 0; r < p.world; ++r) {          // fixed order 0..world-1: bit-identical on every rank
    uint4 v[RED_U];
#pragma unroll
    for (int k = 0; k < RED_U; ++k) {
      v[k] = make_uint4(0, 0, 0, 0);
      if (vi[k] < len) v[k] = (r == p.rank) ? own[vi[k]] : __ldcg(stg + static_cast<size_t>(r) * per + vi[k]);
    }
#pragma unroll
    for (int k = 0; k < RED_U; ++k) acc8<kBF16>(a[k], v[k]);
  }
#pragma unroll
  for (int k = 0; k < RED_U; ++k) {
    if (vi[k] >= len) continue;
    uint4 o;
    o.x = Elem<kBF16>::pack(a[k][0] * p.scale, a[k][1] * p.scale);
    o.y = Elem<kBF16>::pack(a[k][2] * p.scale, a[k][3] * p.scale);
    o.z = Elem<kBF16>::pack(a[k][4] * p.scale, a[k][5] * p.scale);
    o.w = Elem<kBF16>::pack(a[k][6] * p.scale, a[k][7] * p.scale);
    for (int j = 0; j < p.world; ++j) {
      const int q = (p.rank + j) % p.world;
      reinterpret_cast<uint4*>(p.buf[q] + p.byte_offset)[v_lo + vi[k]] = o;
    }
  }
  __syncthreads();
  if (tid == 0) {
    __threadfence_system();
    if (atomicAdd(mine + PF_ARRIVE_C, 1u) == gridDim.x - 1) {
      mine[PF_ARRIVE_C] = 0;
      __threadfence_system();
      for (int q = 0; q < p.world; ++q) st_release_sys(p.flags[q] + PF_BCAST + p.rank, epoch);
      for (int q = 0; q < p.world; ++q) peer_wait(mine, PF_BCAST + q, epoch, 2, p.timeout_cycles);
      mine[PF_EPOCH] = epoch;
      __threadfence_system();
    }
  }
}

// ------------------------------------------------------------------------------------------------
// Form 3 (max_ctas < 0), the default: the COPY ENGINES move the bytes, the SMs only reduce.
// With either SM form, issuing the exchange slice by slice during the backward gains little over
// issuing it once after the backward — exchange CTAs that are
// scheduled ahead of the backward's CTAs stall it, exchange CTAs scheduled behind them do not run
// until it is over.  So the SMs are taken out of the data path:
//   A  (world-1) cudaMemcpyAsync nodes: my sub-slice q  ->  stage_q[rank]          (DMA over NVLink)
//      peer_sync_kernel<1>  (1 CTA, 32 threads): PUSH signals / waits
//   C  peer_reduce_local_kernel: own sub-slice + staged copies -> own arena          (local HBM only)
//      (world-1) cudaMemcpyAsync nodes: reduced sub-slice -> every peer's arena     (DMA over NVLink)
//      peer_sync_kernel<2>: BCAST signals / waits, epoch bump
// Same protocol, same flags, same hazards as above; every node is capturable, so the exchange is still
// part of the step's one CUDA graph, and it shares nothing with the backward but HBM bandwidth.
template <int kPhase>
__global__ void __launch_bounds__(32) peer_sync_kernel(const PeerParams p) {
  uint32_t* mine = p.flags[p.rank];
  const int tid = threadIdx.x;
  const uint32_t epoch = ld_relaxed_sys(mine + PF_EPOCH) + 1u;
  const int word = (kPhase == 1) ? PF_PUSH : PF_BCAST;
  if (tid < p.world) {
    __threadfence_system();
    st_release_sys(p.flags[tid] + word + p.rank, epoch);
    peer_wait(mine, word + tid, epoch, kPhase, p.timeout_cycles);
  }
  __syncwarp();
  if (kPhase == 2 && tid == 0) {
    mine[PF_EPOCH] = epoch;
    __threadfence_system();
  }
}

template <bool kBF16>
__global__ void __launch_bounds__(256, 4) peer_reduce_local_kernel(const PeerParams p) {
  const int tid = threadIdx.x;
  const uint32_t per = static_cast<uint32_t>(p.per), nvec = static_cast<uint32_t>(p.nvec);
  const uint32_t v_lo = static_cast<uint32_t>(p.rank) * per;
  const uint32_t len = (v_lo < nvec) ? min(per, nvec - v_lo) : 0u;
  uint4* own = reinterpret_cast<uint4*>(p.buf[p.rank] + p.byte_offset) + v_lo;
  const uint4* stg = reinterpret_cast<const uint4*>(p.stage[p.rank]);
  float a[RED_U][8];
  uint32_t vi[RED_U];
#pragma unroll
  for (int k = 0; k < RED_U; ++k) {
    vi[k] = blockIdx.x * RED_VPC + k * 256 + tid;
#pragma unroll
    for (int i = 0; i < 8; ++i) a[k][i] = 0.f;
  }
  for (int r = 0; r < p.world; ++r) {          // fixed order 0..world-1
    uint4 v[RED_U];
#pragma unroll
    for (int k = 0; k < RED_U; ++k) {
      v[k] = make_uint4(0, 0, 0, 0);
      if (vi[k] < len) v[k] = (r == p.rank) ? own[vi[k]] : __ldcg(stg + static_cast<size_t>(r) * per + vi[k]);
    }
#pragma unroll
    for (int k = 0; k < RED_U; ++k) acc8<kBF16>(a[k], v[k]);
  }
#pragma unroll
  for (int k = 0; k < RED_U; ++k) {
    if (vi[k] >= len) continue;
    uint4 o;
    o.x = Elem<kBF16>::pack(a[k][0] * p.scale, a[k][1] * p.scale);
    o.y = Elem<kBF16>::pack(a[k][2] * p.scale, a[k][3] * p.scale);
    o.z = Elem<kBF16>::pack(a[k][4] * p.scale, a[k][5] * p.scale);
    o.w = Elem<kBF16>::pack(a[k][6] * p.scale, a[k][7] * p.scale);
    own[vi[k]] = o;
  }
}

static PFN_cuMemGetAddressRange_v3020 get_addr_range() {
  static PFN_cuMemGetAddressRange_v3020 fn = nullptr;
  if (fn == nullptr) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuMemGetAddressRange", &p, cudaEnableDefault, &q) == cudaSuccess &&
        q == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<PFN_cuMemGetAddressRange_v3020>(p);
  }
  return fn;
}

}  // namespace ub

extern "C" {

int64_t ub200_peer_flags_bytes(void) { return ub::PF_WORDS * 4; }

int64_t ub200_peer_stage_bytes(int64_t count, int32_t world) {
  if (count <= 0 || world < 1) return 0;
  const int64_t nvec = (count + 7) / 8;
  int64_t per = (nvec + world - 1) / world;
  per = (per + ub::PUSH_VPC - 1) / ub::PUSH_VPC * ub::PUSH_VPC;
  return per * world * 16;
}

int ub200_peer_ipc_export(const void* dev_ptr, void* handle64, int64_t* offset_bytes) {
  UB_CHECK_ARG(dev_ptr && handle64 && offset_bytes, "peer_ipc_export: null argument");
  auto fn = ub::get_addr_range();
  if (fn == nullptr) return ub::set_error(UB200_ECUDA, "cuMemGetAddressRange entry point unavailable");
  CUdeviceptr base = 0;
  size_t size = 0;
  CUresult r = fn(&base, &size, reinterpret_cast<CUdeviceptr>(dev_ptr));
  if (r != CUDA_SUCCESS) return ub::set_error(UB200_ECUDA, "cuMemGetAddressRange failed (%d)", (int)r);
  cudaIpcMemHandle_t h;
  UB_CHECK_CUDA(cudaIpcGetMemHandle(&h, reinterpret_cast<void*>(base)));
  static_assert(sizeof(h) == 64, "cudaIpcMemHandle_t is 64 bytes");
  memcpy(handle64, &h, 64);
  *offset_bytes = static_cast<int64_t>(reinterpret_cast<CUdeviceptr>(dev_ptr) - base);
  return 0;
}

int ub200_peer_ipc_open(const void* handle64, void** mapped_base) {
  UB_CHECK_ARG(handle64 && mapped_base, "peer_ipc_open: null argument");
  cudaIpcMemHandle_t h;
  memcpy(&h, handle64, 64);
  void* p = nullptr;
  UB_CHECK_CUDA(cudaIpcOpenMemHandle(&p, h, cudaIpcMemLazyEnablePeerAccess));
  *mapped_base = p;
  return 0;
}

int ub200_peer_ipc_close(void* mapped_base) {
  UB_CHECK_ARG(mapped_base, "peer_ipc_close: null argument");
  UB_CHECK_CUDA(cudaIpcCloseMemHandle(mapped_base));
  return 0;
}

int ub200_peer_allreduce(const ub200_peer_allreduce_args* a, ub200_stream_t stream) {
  UB_CHECK_ARG(a, "peer_allreduce: null args");
  UB_CHECK_ARG(a->world >= 1 && a->world <= UB200_MAX_PEERS && a->rank >= 0 && a->rank < a->world,
               "peer_allreduce: rank %d / world %d", a->rank, a->world);
  UB_CHECK_ARG(a->dtype == UB200_F16 || a->dtype == UB200_BF16, "peer_allreduce: dtype");
  UB_CHECK_ARG(a->offset >= 0 && a->count >= 0 && a->offset % 8 == 0 && a->count % 8 == 0,
               "peer_allreduce: offset / count must be multiples of 8 elements (16 bytes)");
  if (a->count == 0) return 0;
  ub::PeerParams p{};
  for (int q = 0; q < a->world; ++q) {
    UB_CHECK_ARG(a->buf[q] && a->stage[q] && a->flags[q], "peer_allreduce: null pointer for rank %d", q);
    UB_CHECK_ARG((reinterpret_cast<uintptr_t>(a->buf[q]) & 15) == 0 &&
                     (reinterpret_cast<uintptr_t>(a->stage[q]) & 15) == 0,
                 "peer_allreduce: buffers must be 16-byte aligned");
    p.buf[q] = static_cast<uint8_t*>(a->buf[q]);
    p.stage[q] = static_cast<uint8_t*>(a->stage[q]);
    p.flags[q] = a->flags[q];
  }
  p.rank = a->rank;
  p.world = a->world;
  p.byte_offset = a->offset * 2;
  p.nvec = a->count / 8;
  long long per = (p.nvec + a->world - 1) / a->world;
  per = (per + ub::PUSH_VPC - 1) / ub::PUSH_VPC * ub::PUSH_VPC;   // whole push CTAs (and whole warp chunks)
  p.per = per;
  UB_CHECK_ARG(per * a->world < (1ll << 31), "peer_allreduce: slice too large (%lld vectors)", (long long)p.nvec);
  UB_CHECK_ARG(per * a->world * 16 <= a->stage_bytes,
               "peer_allreduce: staging buffer too small (%lld < %lld bytes)", (long long)a->stage_bytes,
               (long long)(per * a->world * 16));
  p.scale = a->scale;
  // flag waits count SM clocks: convert at the device's maximum SM clock (a slower clock only
  // lengthens the bound)
  int clock_khz = 0, dev = 0;
  UB_CHECK_CUDA(cudaGetDevice(&dev));
  UB_CHECK_CUDA(cudaDeviceGetAttribute(&clock_khz, cudaDevAttrClockRate, dev));
  p.timeout_cycles = static_cast<long long>(a->timeout_ms > 0 ? a->timeout_ms : 20000) * clock_khz;
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  if (a->max_ctas < 0) {
    // form 3: copy engines for the NVLink transfers, SMs for the flags and the local reduction
    const long long v_lo = p.rank * per;
    long long len = p.nvec - v_lo;
    if (len > per) len = per;
    if (len < 0) len = 0;
    for (int j = 0; j + 1 < a->world; ++j) {
      const int q = (p.rank + 1 + j) % a->world;
      long long q_len = p.nvec - static_cast<long long>(q) * per;
      if (q_len > per) q_len = per;
      if (q_len > 0)
        UB_CHECK_CUDA(cudaMemcpyAsync(p.stage[q] + static_cast<size_t>(p.rank) * per * 16,
                                      p.buf[p.rank] + p.byte_offset + static_cast<size_t>(q) * per * 16,
                                      static_cast<size_t>(q_len) * 16, cudaMemcpyDeviceToDevice, s));
    }
    {
      ub::ProfScope prof(s);
      ub::peer_sync_kernel<1><<<1, 32, 0, s>>>(p);
    }
    if (len > 0) {
      const unsigned gc = static_cast<unsigned>((len + ub::RED_VPC - 1) / ub::RED_VPC);
      ub::ProfScope prof(s);
      if (a->dtype == UB200_BF16) ub::peer_reduce_local_kernel<true><<<gc, 256, 0, s>>>(p);
      else ub::peer_reduce_local_kernel<false><<<gc, 256, 0, s>>>(p);
      for (int j = 0; j + 1 < a->world; ++j) {
        const int q = (p.rank + 1 + j) % a->world;
        UB_CHECK_CUDA(cudaMemcpyAsync(p.buf[q] + p.byte_offset + static_cast<size_t>(v_lo) * 16,
                                      p.buf[p.rank] + p.byte_offset + static_cast<size_t>(v_lo) * 16,
                                      static_cast<size_t>(len) * 16, cudaMemcpyDeviceToDevice, s));
      }
    }
    {
      ub::ProfScope prof(s);
      ub::peer_sync_kernel<2><<<1, 32, 0, s>>>(p);
    }
    UB_CHECK_CUDA(cudaGetLastError());
    return 0;
  }
  if (a->max_ctas == 0) {
    // form 2: work-sized grids of short-lived CTAs (push kernel, then reduce kernel)
    if (a->world > 1) {
      ub::ProfScope prof(s);
      ub::peer_push_kernel<<<dim3(static_cast<unsigned>(per / ub::PUSH_VPC), a->world - 1), 256, 0, s>>>(p);
      UB_CHECK_CUDA(cudaGetLastError());
    }
    const long long v_lo = p.rank * per;
    long long len = p.nvec - v_lo;
    if (len > per) len = per;
    if (len < 0) len = 0;
    const unsigned gc = static_cast<unsigned>((len + ub::RED_VPC - 1) / ub::RED_VPC);
    ub::ProfScope prof(s);
    if (a->dtype == UB200_BF16)
      ub::peer_reduce_kernel<true><<<gc < 1 ? 1 : gc, 256, 0, s>>>(p);
    else
      ub::peer_reduce_kernel<false><<<gc < 1 ? 1 : gc, 256, 0, s>>>(p);
    UB_CHECK_CUDA(cudaGetLastError());
    return 0;
  }
  int ctas = a->max_ctas;
  const long long chunks = per / 32;
  const long long want = (chunks * (a->world > 1 ? a->world - 1 : 1) + 7) / 8;   // >= 1 warp-round per CTA
  if (ctas > want) ctas = static_cast<int>(want < 1 ? 1 : want);
  if (ctas > ub::num_sms()) ctas = ub::num_sms();
  ub::ProfScope prof(s);
  if (a->dtype == UB200_BF16)
    ub::peer_allreduce_kernel<true><<<ctas, 256, 0, s>>>(p);
  else
    ub::peer_allreduce_kernel<false><<<ctas, 256, 0, s>>>(p);
  UB_CHECK_CUDA(cudaGetLastError());
  return 0;
}

}  // extern "C"
