// peer.cu -- the one exchange step of the hot path (SURVEY 8e): an all-gather of the fixed-size per-image
// detection record across the GPUs of one NVSwitch box, done by the ranks themselves over peer memory.
//
// Every rank owns one "mailbox" allocation (cudaMalloc, exported with CUDA IPC and mapped by every peer):
//
//   data  [n_slots][4 parities][world][rec_floats]   records as they arrive from each rank
//   flags [n_slots][world]                           sequence number of the newest record of (slot, rank)
//   seq   [n_slots]                                   this rank's own step counter per slot (device-resident, so
//                                                     that put/wait can be captured into a CUDA graph and replayed)
//
// put  : CTA p stores the local record into rank p's mailbox with 128-bit stores over NVLink (P2P writes are
//        posted: no round trip), fences at system scope, then releases that peer's flag.  40 KB per peer.
// wait : CTA q acquires flag (slot, q) of the LOCAL mailbox, then copies rank q's record out of the mailbox into
//        the caller's gathered tensor.  The spin is bounded (%globaltimer) so that a lost peer cannot hang the GPU.
//
// Four buffers ("parities", step & 3) per slot make the mailbox safe without an acknowledgement, also when the
// consumer runs `lag` = 1 step behind the producers (put step s, then collect step s-1: no rank ever blocks on a
// slower peer's CURRENT step, only on its previous one): a rank passes its wait for step t only after every peer has
// put step t-1, which each issues (stream order) before copying out step t-2 -- so while a peer still reads t-2 the
// fastest rank can have written at most t+1: four live records.  NCCL stays the control plane (rendezvous, handle
// exchange, barriers).
//
// Counters are 32-bit and compared modulo 2^32 (flags as a signed distance, the early exit unsigned), so the exchange
// runs straight through 2^31.  A slot's counter after 2^32 puts is 0 again, which is also the "nothing put yet" state:
// the wait of that step (and, at lag 1, of the next one too) returns without copying, and the exchange continues
// after it (2^32 is a multiple of the 4 parities).  So 2^32 - 1 steps per slot is the limit of an uninterrupted
// exchange: about 80 days of one slot at 600 steps/s.
#include "common.cuh"

namespace {

constexpr int kMaxPeers = 16;
constexpr int kParities = 4;

struct PeerPtrs {
    float* p[kMaxPeers];
};

__device__ __forceinline__ void st_release_sys(unsigned* p, unsigned v) {
    asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ unsigned ld_acquire_sys(const unsigned* p) {
    unsigned v;
    asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ unsigned long long gtime_ns() {
    unsigned long long t;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t)::"memory");
    return t;
}

struct Layout {
    int n_slots, world, rec_floats;     // rec_floats % 4 == 0
    __host__ __device__ size_t data_floats() const { return (size_t)n_slots * kParities * world * rec_floats; }
    __host__ __device__ size_t data_off(int slot, int par, int r) const {
        return (((size_t)slot * kParities + par) * world + r) * rec_floats;
    }
    __host__ __device__ size_t flag_off(int slot, int r) const { return (size_t)slot * world + r; }   // in u32 after data
    __host__ __device__ size_t seq_off(int slot) const { return (size_t)n_slots * world + slot; }
    __host__ __device__ size_t ticket_off(int slot) const { return (size_t)n_slots * world + n_slots + slot; }
    __host__ __device__ size_t bytes() const { return data_floats() * 4 + ((size_t)n_slots * world + 2 * n_slots) * 4 + 64; }
};

// grid = world CTAs of 256 threads (small enough to co-reside with the 225 KB / 320-thread conv CTAs that fill the
// SMs): CTA p writes the record into rank p's mailbox.  Every CTA reads the slot's step counter before the last one
// to finish (ticket) advances it.
__global__ void __launch_bounds__(256)
peer_put_kernel(const float* __restrict__ rec, PeerPtrs peers, Layout L, int rank, int slot) {
    unsigned* my_ctl = reinterpret_cast<unsigned*>(peers.p[rank] + L.data_floats());
    const int p = blockIdx.x;
    const unsigned seq = my_ctl[L.seq_off(slot)] + 1u;
    const int par = (int)(seq % kParities);
    const int n4 = L.rec_floats / 4;
    const float4* src = reinterpret_cast<const float4*>(rec);
    float4* dst = reinterpret_cast<float4*>(peers.p[p] + L.data_off(slot, par, rank));
    for (int i = threadIdx.x; i < n4; i += blockDim.x) dst[i] = src[i];
    __threadfence_system();
    __syncthreads();
    if (threadIdx.x == 0) {
        unsigned* ctl = reinterpret_cast<unsigned*>(peers.p[p] + L.data_floats());
        st_release_sys(ctl + L.flag_off(slot, rank), seq);
        if (atomicAdd(&my_ctl[L.ticket_off(slot)], 1u) == (unsigned)L.world - 1u) {      // last CTA of this put
            my_ctl[L.ticket_off(slot)] = 0u;
            __threadfence();
            my_ctl[L.seq_off(slot)] = seq;
        }
    }
}

__global__ void __launch_bounds__(128)
peer_wait_kernel(float* __restrict__ mailbox, Layout L, int slot, int lag, float* __restrict__ out, int* __restrict__ err,
                 unsigned long long timeout_ns) {
    const int q = blockIdx.x;
    unsigned* ctl = reinterpret_cast<unsigned*>(mailbox + L.data_floats());
    __shared__ unsigned s_seq;
    __shared__ int s_ok;
    const unsigned cur = ctl[L.seq_off(slot)];          // written by this rank's put (stream order)
    if (cur < 1u + (unsigned)lag) return;               // nothing that old has been put yet (first `lag` calls): CTA-uniform
    if (threadIdx.x == 0) {
        const unsigned seq = cur - (unsigned)lag;
        const unsigned long long t0 = gtime_ns();
        int ok = 1;
        while ((int)(ld_acquire_sys(ctl + L.flag_off(slot, q)) - seq) < 0) {
            if (gtime_ns() - t0 > timeout_ns) { ok = 0; break; }
            __nanosleep(200);
        }
        s_seq = seq;
        s_ok = ok;
        if (!ok) atomicExch(err, 1 + q);
    }
    __syncthreads();
    if (!s_ok) return;
    const int par = (int)(s_seq % kParities);
    const float4* src = reinterpret_cast<const float4*>(mailbox + L.data_off(slot, par, q));
    float4* dst = reinterpret_cast<float4*>(out + (size_t)q * L.rec_floats);
    for (int i = threadIdx.x; i < L.rec_floats / 4; i += blockDim.x) dst[i] = __ldcg(src + i);
}

Layout make_layout(int n_slots, int world, int rec_floats) {
    Layout L;
    L.n_slots = n_slots; L.world = world; L.rec_floats = rec_floats;
    return L;
}

bool misaligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) != 0; }

// the longest wait whose nanosecond count still fits the kernel's u64
constexpr double kMaxTimeoutS = 1.8e10;

}  // namespace

extern "C" size_t sb_peer_mailbox_bytes(int n_slots, int world, int rec_floats) {
    if (n_slots < 1 || world < 1 || world > kMaxPeers || rec_floats < 4 || (rec_floats & 3)) return 0;
    return make_layout(n_slots, world, rec_floats).bytes();
}

extern "C" int sb_peer_alloc(size_t bytes, void** ptr) {
    if (!ptr || bytes == 0) return SB_EINVAL;
    cudaError_t e = cudaMalloc(ptr, bytes);
    if (e != cudaSuccess) return (int)e;
    e = cudaMemset(*ptr, 0, bytes);
    if (e != cudaSuccess) return (int)e;
    return (int)cudaDeviceSynchronize();
}

extern "C" int sb_peer_free(void* ptr) { return (int)cudaFree(ptr); }

extern "C" int sb_ipc_export(void* ptr, void* handle64) {
    static_assert(sizeof(cudaIpcMemHandle_t) == 64, "CUDA IPC handle size");
    if (!ptr || !handle64) return SB_EINVAL;
    return (int)cudaIpcGetMemHandle(reinterpret_cast<cudaIpcMemHandle_t*>(handle64), ptr);
}

extern "C" int sb_ipc_import(const void* handle64, void** ptr) {
    if (!ptr || !handle64) return SB_EINVAL;
    cudaIpcMemHandle_t h;
    memcpy(&h, handle64, sizeof(h));
    return (int)cudaIpcOpenMemHandle(ptr, h, cudaIpcMemLazyEnablePeerAccess);
}

extern "C" int sb_ipc_close(void* ptr) { return (int)cudaIpcCloseMemHandle(ptr); }

extern "C" int sb_peer_put_record(const float* rec, void* const* mailboxes, int n_slots, int world, int rec_floats,
                                  int rank, int slot, sb_stream_t stream) {
    if (!rec || !mailboxes || world < 1 || world > kMaxPeers || rank < 0 || rank >= world || slot < 0 || slot >= n_slots ||
        rec_floats < 4 || (rec_floats & 3) || misaligned16(rec))
        return SB_EINVAL;
    for (int i = 0; i < world; ++i)
        if (!mailboxes[i] || misaligned16(mailboxes[i])) return SB_EINVAL;
    PeerPtrs pp;
    for (int i = 0; i < kMaxPeers; ++i) pp.p[i] = i < world ? static_cast<float*>(mailboxes[i]) : nullptr;
    peer_put_kernel<<<world, 256, 0, sb_cs(stream)>>>(rec, pp, make_layout(n_slots, world, rec_floats), rank, slot);
    SB_LAUNCHED();
    SB_CHECK_LAUNCH();
    return SB_OK;
}

extern "C" int sb_peer_wait_records(void* mailbox, int n_slots, int world, int rec_floats, int slot, int lag,
                                    float* gathered, int* err_flag, double timeout_s, sb_stream_t stream) {
    if (!mailbox || !gathered || !err_flag || world < 1 || world > kMaxPeers || slot < 0 || slot >= n_slots || lag < 0 || lag > 1 ||
        rec_floats < 4 || (rec_floats & 3) || misaligned16(mailbox) || misaligned16(gathered) ||
        !(timeout_s >= 0.0 && timeout_s <= kMaxTimeoutS))                 // also refuses NaN
        return SB_EINVAL;
    peer_wait_kernel<<<world, 128, 0, sb_cs(stream)>>>(static_cast<float*>(mailbox), make_layout(n_slots, world, rec_floats),
                                                       slot, lag, gathered, err_flag,
                                                       (unsigned long long)(timeout_s * 1e9));
    SB_LAUNCHED();
    SB_CHECK_LAUNCH();
    return SB_OK;
}
