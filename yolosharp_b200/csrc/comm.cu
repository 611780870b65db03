// yb_comm: all-gather of small fixed-capacity payloads (the post-NMS detections of every rank) over NVLink peer
// memory, without a collective kernel on the critical path.
//
// Design target: SURVEY.md section 8(e) - "forward + NMS locally into fixed-capacity (B_local, 300, 6[+32]) +
// counts buffers, then one all-gather so every rank holds all detections in image order".  The reference has no
// counterpart (Data/Config.cs:301: single device).  ncclAllGather is a rendezvous: its kernel must be co-resident
// on all ranks to make progress, and on a GPU whose SMs are held by persistent forward kernels it starves.  Here every rank PUSHES its payload into a window of every peer
// with plain stores through peer-mapped pointers (cudaIpc), then publishes a sequence number per (slot, source);
// consumers poll flags in their OWN memory.  No rank ever waits inside a kernel for a peer's kernel to be scheduled
// at the same time.
//
//   window of rank r (one cudaMalloc, exported with cudaIpcGetMemHandle):
//     data  [slots][world][bytes_per_rank]   payload of source s for slot k at (k*world + s)
//     flags [slots][world] u32               sequence number published by source s after its payload landed
//     acks  [slots][world] u32               sequence number up to which CONSUMER s has released slot k of ITS
//                                            window (flow control: a source must not overwrite unread data)
//   send  [slots][bytes_per_rank]            local staging the producer kernel (yb_nms) writes into
//
//   allgather(slot), use number u = 1, 2, ...:
//     push kernel   one CTA per destination p: wait acks[slot][p] >= u-1 (p released the previous contents), copy
//                   send[slot] -> data_p[slot][rank] with 16-byte stores, __threadfence_system, flags_p[slot][rank] = u
//     wait kernel   one thread per source s: spin until flags[slot][s] >= u (own memory)
//   release(slot):  acks_p[slot][rank] = u for every p (after the consumer - a D2H copy, a kernel - is done)
//
// Every spin is bounded (trap after ~10 s) so that a protocol bug cannot hang the GPU.
#include <cstring>
#include <memory>
#include <vector>

#include "common.cuh"

namespace yb {

constexpr int COMM_MAX_WORLD = 16;
constexpr int COMM_MAX_SLOTS = 8;

struct CommDev {
  int rank, world;
  unsigned long long bytes;          // payload bytes per rank, multiple of 16
  char* data[COMM_MAX_WORLD];        // window data section of every rank (peer-mapped)
  unsigned* flags[COMM_MAX_WORLD];
  unsigned* acks[COMM_MAX_WORLD];
};

__device__ __forceinline__ unsigned ld_acquire_sys(const unsigned* p) {
  unsigned v;
  asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void st_release_sys(unsigned* p, unsigned v) {
  asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ void spin_until_ge(const unsigned* p, unsigned want) {
  const long long t0 = clock64();
  while ((int)(ld_acquire_sys(p) - want) < 0) {
    __nanosleep(64);
    if (clock64() - t0 > 20000000000ll) __trap();  // ~10 s: a peer died or the protocol is broken
  }
}

__global__ void __launch_bounds__(512) comm_push_kernel(CommDev c, int slot, const int4* __restrict__ src, unsigned use) {
  const int p = blockIdx.x;
  if (threadIdx.x == 0) spin_until_ge(c.acks[c.rank] + slot * c.world + p, use - 1);
  __syncthreads();
  int4* dst = reinterpret_cast<int4*>(c.data[p] + (size_t)(slot * c.world + c.rank) * c.bytes);
  const int n16 = (int)(c.bytes >> 4);
  for (int i = threadIdx.x; i < n16; i += blockDim.x) dst[i] = src[i];
  __threadfence_system();
  __syncthreads();
  if (threadIdx.x == 0) st_release_sys(c.flags[p] + slot * c.world + c.rank, use);
}

__global__ void comm_wait_kernel(CommDev c, int slot, unsigned use) {
  if ((int)threadIdx.x < c.world) spin_until_ge(c.flags[c.rank] + slot * c.world + threadIdx.x, use);
}

__global__ void comm_release_kernel(CommDev c, int slot, unsigned use) {
  if ((int)threadIdx.x < c.world) st_release_sys(c.acks[threadIdx.x] + slot * c.world + c.rank, use);
}

}  // namespace yb

using namespace yb;

struct yb_comm {
  CommDev dev;
  int device = 0, slots = 0;
  size_t window_bytes = 0, data_bytes = 0;
  char* window = nullptr;  // local window (cudaMalloc base, IPC-exported)
  char* send = nullptr;
  void* peer_base[COMM_MAX_WORLD] = {};  // cudaIpcOpenMemHandle results (nullptr for self)
  unsigned use[COMM_MAX_SLOTS] = {};
  bool connected = false;
};

extern "C" {

int32_t yb_comm_handle_bytes(void) { return (int32_t)sizeof(cudaIpcMemHandle_t); }

int32_t yb_comm_create(int32_t rank, int32_t world, int32_t device, int64_t bytes_per_rank, int32_t slots, yb_comm** out) {
  if (!out) { set_error("yb_comm_create: null argument"); return YB_ERR_INVALID_ARG; }
  *out = nullptr;
  if (world < 1 || world > COMM_MAX_WORLD || rank < 0 || rank >= world) { set_error("yb_comm_create: need 0 <= rank < world <= 16"); return YB_ERR_INVALID_ARG; }
  if (slots < 1 || slots > COMM_MAX_SLOTS) { set_error("yb_comm_create: slots outside [1,8]"); return YB_ERR_INVALID_ARG; }
  if (bytes_per_rank <= 0 || bytes_per_rank % 16 || bytes_per_rank > (1ll << 30)) { set_error("yb_comm_create: bytes_per_rank must be a positive multiple of 16 (<= 1 GiB)"); return YB_ERR_INVALID_ARG; }
  int ndev = 0;
  if (!have_device("yb_comm_create", &ndev)) return YB_ERR_NO_DEVICE;
  if (device < 0 || device >= ndev) { set_error("yb_comm_create: bad device ordinal"); return YB_ERR_INVALID_ARG; }
  YB_CUDA_CHECK(cudaSetDevice(device));
  std::unique_ptr<yb_comm> c(new yb_comm());
  c->device = device;
  c->slots = slots;
  c->dev.rank = rank; c->dev.world = world; c->dev.bytes = (unsigned long long)bytes_per_rank;
  c->data_bytes = (size_t)slots * world * bytes_per_rank;
  const size_t flag_bytes = ((size_t)slots * world * sizeof(unsigned) + 255) / 256 * 256;
  c->window_bytes = c->data_bytes + 2 * flag_bytes;
  YB_CUDA_CHECK(cudaMalloc((void**)&c->window, c->window_bytes));
  YB_CUDA_CHECK(cudaMemset(c->window, 0, c->window_bytes));
  YB_CUDA_CHECK(cudaMalloc((void**)&c->send, (size_t)slots * bytes_per_rank));
  YB_CUDA_CHECK(cudaMemset(c->send, 0, (size_t)slots * bytes_per_rank));
  YB_CUDA_CHECK(cudaDeviceSynchronize());
  *out = c.release();
  return YB_OK;
}

int32_t yb_comm_local_handle(yb_comm* c, void* handle_out) {
  if (!c || !handle_out) { set_error("yb_comm_local_handle: null argument"); return YB_ERR_INVALID_ARG; }
  YB_CUDA_CHECK(cudaSetDevice(c->device));
  cudaIpcMemHandle_t h;
  YB_CUDA_CHECK(cudaIpcGetMemHandle(&h, c->window));
  std::memcpy(handle_out, &h, sizeof(h));
  return YB_OK;
}

int32_t yb_comm_connect(yb_comm* c, const void* handles) {
  if (!c || !handles) { set_error("yb_comm_connect: null argument"); return YB_ERR_INVALID_ARG; }
  if (c->connected) { set_error("yb_comm_connect: already connected"); return YB_ERR_STATE; }
  YB_CUDA_CHECK(cudaSetDevice(c->device));
  const size_t flag_bytes = (c->window_bytes - c->data_bytes) / 2;
  for (int p = 0; p < c->dev.world; p++) {
    char* base = c->window;
    if (p != c->dev.rank) {
      cudaIpcMemHandle_t h;
      std::memcpy(&h, (const char*)handles + (size_t)p * sizeof(h), sizeof(h));
      void* ptr = nullptr;
      cudaError_t ce = cudaIpcOpenMemHandle(&ptr, h, cudaIpcMemLazyEnablePeerAccess);
      if (ce != cudaSuccess) {
        set_error(std::string("yb_comm_connect: cudaIpcOpenMemHandle for rank ") + std::to_string(p) + " failed: " +
                  cudaGetErrorString(ce) + " (ranks must be processes on one node with peer access)");
        cudaGetLastError();
        return YB_ERR_CUDA;
      }
      c->peer_base[p] = ptr;
      base = (char*)ptr;
    }
    c->dev.data[p] = base;
    c->dev.flags[p] = reinterpret_cast<unsigned*>(base + c->data_bytes);
    c->dev.acks[p] = reinterpret_cast<unsigned*>(base + c->data_bytes + flag_bytes);
  }
  c->connected = true;
  return YB_OK;
}

int32_t yb_comm_info(const yb_comm* c, int32_t* rank, int32_t* world, int64_t* bytes_per_rank, int32_t* slots) {
  if (!c) { set_error("yb_comm_info: null comm"); return YB_ERR_INVALID_ARG; }
  if (rank) *rank = c->dev.rank;
  if (world) *world = c->dev.world;
  if (bytes_per_rank) *bytes_per_rank = (int64_t)c->dev.bytes;
  if (slots) *slots = c->slots;
  return YB_OK;
}

int64_t yb_comm_detection_payload_bytes(int32_t batch, int32_t max_det, int32_t row_width) {
  const int64_t dets = (int64_t)batch * max_det * row_width * 4;
  return (dets + 15) / 16 * 16 + ((int64_t)batch * 4 + 15) / 16 * 16;
}

void* yb_comm_send_buffer(yb_comm* c, int32_t slot) {
  if (!c || slot < 0 || slot >= c->slots) return nullptr;
  return c->send + (size_t)slot * c->dev.bytes;
}

void* yb_comm_window(yb_comm* c, int32_t slot) {
  if (!c || slot < 0 || slot >= c->slots) return nullptr;
  return c->window + (size_t)slot * c->dev.world * c->dev.bytes;
}

int32_t yb_comm_allgather(yb_comm* c, int32_t slot, void* stream) {
  if (!c || slot < 0 || slot >= c->slots) { set_error("yb_comm_allgather: bad comm / slot"); return YB_ERR_INVALID_ARG; }
  if (!c->connected) { set_error("yb_comm_allgather: call yb_comm_connect first"); return YB_ERR_STATE; }
  YB_CUDA_CHECK(cudaSetDevice(c->device));
  cudaStream_t s = (cudaStream_t)stream;
  const unsigned use = ++c->use[slot];
  comm_push_kernel<<<c->dev.world, 512, 0, s>>>(c->dev, slot, reinterpret_cast<const int4*>(c->send + (size_t)slot * c->dev.bytes), use);
  comm_wait_kernel<<<1, 32, 0, s>>>(c->dev, slot, use);
  YB_CUDA_CHECK(cudaGetLastError());
  return YB_OK;
}

int32_t yb_comm_release(yb_comm* c, int32_t slot, void* stream) {
  if (!c || slot < 0 || slot >= c->slots) { set_error("yb_comm_release: bad comm / slot"); return YB_ERR_INVALID_ARG; }
  if (!c->connected || c->use[slot] == 0) { set_error("yb_comm_release: nothing gathered on this slot"); return YB_ERR_STATE; }
  YB_CUDA_CHECK(cudaSetDevice(c->device));
  comm_release_kernel<<<1, 32, 0, (cudaStream_t)stream>>>(c->dev, slot, c->use[slot]);
  YB_CUDA_CHECK(cudaGetLastError());
  return YB_OK;
}

void yb_comm_destroy(yb_comm* c) {
  if (!c) return;
  cudaSetDevice(c->device);
  cudaDeviceSynchronize();
  for (int p = 0; p < c->dev.world; p++)
    if (c->peer_base[p]) cudaIpcCloseMemHandle(c->peer_base[p]);
  if (c->window) cudaFree(c->window);
  if (c->send) cudaFree(c->send);
  delete c;
}

}  // extern "C"
