// Capability + bandwidth probe for the B200 peer-memory transport.
// Forks one process per GPU; parent relays messages/fds (star topology).
// Build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o tools/probe tools/probe.cu -lcuda
// Run:   tools/probe <ngpus> [isolate]
#include <cuda.h>
#include <cuda_runtime.h>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <cstdint>
#include <vector>
#include <string>
#include <unistd.h>
#include <sys/socket.h>
#include <sys/wait.h>
#include <sys/uio.h>
#include <errno.h>

#define CK(x) do { cudaError_t e_ = (x); if (e_ != cudaSuccess) { printf("[r%d] CUDA error %s at %s:%d: %s\n", g_rank, #x, __FILE__, __LINE__, cudaGetErrorString(e_)); fflush(stdout); return -1; } } while (0)
#define CU(x) do { CUresult e_ = (x); if (e_ != CUDA_SUCCESS) { const char* s_=nullptr; cuGetErrorString(e_, &s_); printf("[r%d] CU error %s at %s:%d: %d %s\n", g_rank, #x, __FILE__, __LINE__, (int)e_, s_?s_:"?"); fflush(stdout); return -1; } } while (0)

static int g_rank = -1, g_world = 0, g_sock = -1, g_exp = 0;

// ---------- message passing with optional fd ----------
static int send_msg(int sock, const void* buf, size_t len, int fd) {
  struct msghdr msg = {}; struct iovec iov; char cbuf[CMSG_SPACE(sizeof(int))];
  uint64_t hdr = len;
  iov.iov_base = &hdr; iov.iov_len = sizeof(hdr);
  msg.msg_iov = &iov; msg.msg_iovlen = 1;
  if (fd >= 0) {
    memset(cbuf, 0, sizeof(cbuf));
    msg.msg_control = cbuf; msg.msg_controllen = sizeof(cbuf);
    struct cmsghdr* c = CMSG_FIRSTHDR(&msg);
    c->cmsg_level = SOL_SOCKET; c->cmsg_type = SCM_RIGHTS; c->cmsg_len = CMSG_LEN(sizeof(int));
    memcpy(CMSG_DATA(c), &fd, sizeof(int));
  }
  if (sendmsg(sock, &msg, 0) != (ssize_t)sizeof(hdr)) return -1;
  size_t off = 0;
  while (off < len) { ssize_t n = write(sock, (const char*)buf + off, len - off); if (n <= 0) return -1; off += n; }
  return 0;
}
static int recv_msg(int sock, std::string& out, int* fd_out) {
  struct msghdr msg = {}; struct iovec iov; char cbuf[CMSG_SPACE(sizeof(int))];
  uint64_t hdr = 0;
  iov.iov_base = &hdr; iov.iov_len = sizeof(hdr);
  msg.msg_iov = &iov; msg.msg_iovlen = 1; msg.msg_control = cbuf; msg.msg_controllen = sizeof(cbuf);
  ssize_t n = recvmsg(sock, &msg, MSG_WAITALL);
  if (n != (ssize_t)sizeof(hdr)) return -1;
  *fd_out = -1;
  for (struct cmsghdr* c = CMSG_FIRSTHDR(&msg); c; c = CMSG_NXTHDR(&msg, c))
    if (c->cmsg_level == SOL_SOCKET && c->cmsg_type == SCM_RIGHTS) memcpy(fd_out, CMSG_DATA(c), sizeof(int));
  out.resize(hdr);
  size_t off = 0;
  while (off < hdr) { ssize_t k = read(sock, &out[off], hdr - off); if (k <= 0) return -1; off += k; }
  return 0;
}
// child side allgather through the parent
static int allgather(const void* buf, size_t len, int fd, std::vector<std::string>& msgs, std::vector<int>& fds) {
  if (send_msg(g_sock, buf, len, fd)) { printf("[r%d] send_msg failed %d\n", g_rank, errno); return -1; }
  msgs.resize(g_world); fds.assign(g_world, -1);
  for (int i = 0; i < g_world; i++) if (recv_msg(g_sock, msgs[i], &fds[i])) { printf("[r%d] recv_msg failed\n", g_rank); return -1; }
  return 0;
}
static int barrier() { std::vector<std::string> m; std::vector<int> f; char c = 0; return allgather(&c, 1, -1, m, f); }

// ---------- kernels ----------
__global__ void fill_kernel(float* p, size_t n, float v) {
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) p[i] = v;
}
__global__ void check_kernel(const float* p, size_t n, float v, unsigned long long* bad) {
  unsigned long long b = 0;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) b += (p[i] != v);
  if (b) atomicAdd(bad, b);
}
template <int UNROLL>
__global__ void __launch_bounds__(512) copy_kernel(uint4* __restrict__ dst, const uint4* __restrict__ src, size_t n16) {
  size_t stride = (size_t)gridDim.x * blockDim.x;
  size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  for (; i + (UNROLL - 1) * stride < n16; i += UNROLL * stride) {
    uint4 v[UNROLL];
#pragma unroll
    for (int u = 0; u < UNROLL; u++) v[u] = src[i + u * stride];
#pragma unroll
    for (int u = 0; u < UNROLL; u++) dst[i + u * stride] = v[u];
  }
  for (; i < n16; i += stride) dst[i] = src[i];
}
// gather 1/W slices from each of W sources (two-shot pull pattern)
struct Ptrs { const uint4* p[8]; };
template <int UNROLL>
__global__ void __launch_bounds__(512) multi_pull_kernel(uint4* __restrict__ dst, Ptrs srcs, int nsrc, size_t n16_per) {
  size_t stride = (size_t)gridDim.x * blockDim.x;
  for (int s = 0; s < nsrc; s++) {
    const uint4* src = srcs.p[s] + (size_t)s * n16_per; uint4* d = dst + (size_t)s * n16_per;
    size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
    for (; i + (UNROLL - 1) * stride < n16_per; i += UNROLL * stride) {
      uint4 v[UNROLL];
#pragma unroll
      for (int u = 0; u < UNROLL; u++) v[u] = src[i + u * stride];
#pragma unroll
      for (int u = 0; u < UNROLL; u++) d[i + u * stride] = v[u];
    }
    for (; i < n16_per; i += stride) d[i] = src[i];
  }
}
__global__ void __launch_bounds__(512) mc_ldreduce_kernel(float4* __restrict__ dst, const float4* mc, size_t n16) {
  size_t stride = (size_t)gridDim.x * blockDim.x;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n16; i += stride) {
    float4 v;
    asm volatile("multimem.ld_reduce.relaxed.sys.global.add.v4.f32 {%0,%1,%2,%3}, [%4];"
                 : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "l"(mc + i) : "memory");
    dst[i] = v;
  }
}
__global__ void __launch_bounds__(512) mc_ldreduce_bf16_kernel(uint4* __restrict__ dst, const uint4* mc, size_t n16) {
  size_t stride = (size_t)gridDim.x * blockDim.x;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n16; i += stride) {
    uint4 v;
    asm volatile("multimem.ld_reduce.relaxed.sys.global.add.acc::f32.v4.bf16x2 {%0,%1,%2,%3}, [%4];"
                 : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(mc + i) : "memory");
    dst[i] = v;
  }
}
__global__ void __launch_bounds__(512) mc_st_kernel(float4* mc, const float4* __restrict__ src, size_t n16) {
  size_t stride = (size_t)gridDim.x * blockDim.x;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n16; i += stride) {
    float4 v = src[i];
    asm volatile("multimem.st.relaxed.sys.global.v4.f32 [%0], {%1,%2,%3,%4};"
                 :: "l"(mc + i), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w) : "memory");
  }
}
// fused: ld_reduce own slice + st broadcast (NVLS allreduce inner loop)
__global__ void __launch_bounds__(512) mc_allreduce_kernel(float4* mc, size_t begin16, size_t n16) {
  size_t stride = (size_t)gridDim.x * blockDim.x;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n16; i += stride) {
    float4 v;
    asm volatile("multimem.ld_reduce.relaxed.sys.global.add.v4.f32 {%0,%1,%2,%3}, [%4];"
                 : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "l"(mc + begin16 + i) : "memory");
    asm volatile("multimem.st.relaxed.sys.global.v4.f32 [%0], {%1,%2,%3,%4};"
                 :: "l"(mc + begin16 + i), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w) : "memory");
  }
}
// ping-pong flag latency: rank0 writes k to peer flag, waits for own flag == k
__global__ void pingpong_kernel(volatile unsigned* my_flag, unsigned* peer_flag, int iters, int first, long long* cycles) {
  long long t0 = clock64();
  for (int k = 1; k <= iters; k++) {
    if (first) {
      asm volatile("st.release.sys.global.u32 [%0], %1;" :: "l"(peer_flag), "r"((unsigned)k) : "memory");
      unsigned v; do { asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(my_flag) : "memory"); } while (v < (unsigned)k);
    } else {
      unsigned v; do { asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(my_flag) : "memory"); } while (v < (unsigned)k);
      asm volatile("st.release.sys.global.u32 [%0], %1;" :: "l"(peer_flag), "r"((unsigned)k) : "memory");
    }
  }
  *cycles = clock64() - t0;
}


// ---------------------------------------------------------------------------------------------
// round-2 experiments (run with: tools/probe <ngpus> exp)
// ---------------------------------------------------------------------------------------------
// E2: CTAs [0, n_nvls) reduce+broadcast through the switch, CTAs [n_nvls, grid) push unicast to peers.
__global__ void __launch_bounds__(512) mix_kernel(float4* mc, size_t nvls_begin16, size_t nvls_n16, int n_nvls,
                                                  Ptrs peers, int rank, int world, const uint4* __restrict__ src,
                                                  size_t p2p_dst_off16, size_t p2p_n16) {
  if ((int)blockIdx.x < n_nvls) {
    size_t stride = (size_t)n_nvls * blockDim.x;
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < nvls_n16; i += stride) {
      float4 v;
      asm volatile("multimem.ld_reduce.relaxed.sys.global.add.v4.f32 {%0,%1,%2,%3}, [%4];"
                   : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "l"(mc + nvls_begin16 + i) : "memory");
      asm volatile("multimem.st.relaxed.sys.global.v4.f32 [%0], {%1,%2,%3,%4};"
                   :: "l"(mc + nvls_begin16 + i), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w) : "memory");
    }
  } else {
    int nb = gridDim.x - n_nvls, b = blockIdx.x - n_nvls;
    size_t per_peer = p2p_n16 / (world - 1);
    for (int k = 1; k < world; k++) {
      int j = (rank + k) % world;
      uint4* dst = (uint4*)peers.p[j] + p2p_dst_off16 + (size_t)rank * per_peer;
      const uint4* s = src + (size_t)(k - 1) * per_peer;
      size_t stride = (size_t)nb * blockDim.x;
      size_t i = b * (size_t)blockDim.x + threadIdx.x;
      for (; i + 3 * stride < per_peer; i += 4 * stride) {
        uint4 v0 = s[i], v1 = s[i + stride], v2 = s[i + 2 * stride], v3 = s[i + 3 * stride];
        dst[i] = v0; dst[i + stride] = v1; dst[i + 2 * stride] = v2; dst[i + 3 * stride] = v3;
      }
      for (; i < per_peer; i += stride) dst[i] = s[i];
    }
  }
}
// E3: cost of a system-scope fence while the other warps of the CTA keep streaming stores to a peer.
__global__ void __launch_bounds__(512) fence_kernel(uint4* peer_dst, const uint4* __restrict__ src, size_t n16, unsigned* peer_flag,
                                                   int iters, int do_stream, long long* cycles_out) {
  __shared__ volatile int done;
  if (threadIdx.x == 0) done = 0;
  __syncthreads();
  if (threadIdx.x < 32) {
    if (threadIdx.x == 0) {
      long long t0 = clock64();
      for (int k = 1; k <= iters; k++) {
        asm volatile("fence.acq_rel.sys;" ::: "memory");
        asm volatile("st.relaxed.sys.global.u32 [%0], %1;" :: "l"(peer_flag + blockIdx.x), "r"((unsigned)k) : "memory");
      }
      long long t1 = clock64();
      if (blockIdx.x == 0) *cycles_out = (t1 - t0) / iters;
      done = 1;
    }
  } else if (do_stream) {
    size_t per = n16 / gridDim.x, base = per * blockIdx.x;
    size_t i = threadIdx.x - 32;
    while (!done) {
      peer_dst[base + i] = src[base + i];
      i += 480; if (i >= per) i = threadIdx.x - 32;
    }
  }
}
// E4: packed data+flag (one 16-byte store, no fence) ping-pong
__global__ void ll_pingpong_kernel(uint4* my_slot, uint4* peer_slot, int iters, int first) {
  for (int k = 1; k <= iters; k++) {
    uint4 out = make_uint4(0xabcd0000u + k, 0x1234u, 0x5678u, (unsigned)k);
    if (first) {
      asm volatile("st.volatile.global.v4.u32 [%0], {%1,%2,%3,%4};" :: "l"(peer_slot), "r"(out.x), "r"(out.y), "r"(out.z), "r"(out.w) : "memory");
      uint4 v; do { asm volatile("ld.volatile.global.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(my_slot) : "memory"); } while (v.w != (unsigned)k);
    } else {
      uint4 v; do { asm volatile("ld.volatile.global.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(my_slot) : "memory"); } while (v.w != (unsigned)k);
      asm volatile("st.volatile.global.v4.u32 [%0], {%1,%2,%3,%4};" :: "l"(peer_slot), "r"(out.x), "r"(out.y), "r"(out.z), "r"(out.w) : "memory");
    }
  }
}

static float time_ms(cudaEvent_t a, cudaEvent_t b) { float ms = 0; cudaEventElapsedTime(&ms, a, b); return ms; }

struct Vmm { CUmemGenericAllocationHandle h; CUdeviceptr va; size_t size; };

static int child_main(int isolate) {
  int dev = isolate ? 0 : g_rank;
  if (isolate) { char b[16]; snprintf(b, sizeof b, "%d", g_rank); setenv("CUDA_VISIBLE_DEVICES", b, 1); }
  CK(cudaSetDevice(dev)); CK(cudaFree(0));
  CU(cuInit(0));
  CUdevice cudev; CU(cuDeviceGet(&cudev, dev));
  cudaDeviceProp prop; CK(cudaGetDeviceProperties(&prop, dev));
  int ndev = 0; cudaGetDeviceCount(&ndev);
  int a_mc = 0, a_fd = 0, a_fab = 0, a_vmm = 0;
  cuDeviceGetAttribute(&a_mc, CU_DEVICE_ATTRIBUTE_MULTICAST_SUPPORTED, cudev);
  cuDeviceGetAttribute(&a_fd, CU_DEVICE_ATTRIBUTE_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR_SUPPORTED, cudev);
  cuDeviceGetAttribute(&a_fab, CU_DEVICE_ATTRIBUTE_HANDLE_TYPE_FABRIC_SUPPORTED, cudev);
  cuDeviceGetAttribute(&a_vmm, CU_DEVICE_ATTRIBUTE_VIRTUAL_MEMORY_MANAGEMENT_SUPPORTED, cudev);
  int drv = 0; cuDriverGetVersion(&drv);
  if (g_rank == 0) {
    printf("PROBE dev=%s sm=%d.%d SMs=%d visible_devices=%d driver=%d mc=%d posix_fd=%d fabric=%d vmm=%d isolate=%d\n",
           prop.name, prop.major, prop.minor, prop.multiProcessorCount, ndev, drv, a_mc, a_fd, a_fab, a_vmm, isolate);
    if (!isolate) for (int j = 1; j < ndev && j < g_world; j++) { int can = 0; cudaDeviceCanAccessPeer(&can, 0, j); printf("PROBE canAccessPeer 0->%d = %d\n", j, can); }
    fflush(stdout);
  }
  const size_t BYTES = 256ull << 20; const size_t NF = BYTES / 4;
  cudaEvent_t e0, e1; CK(cudaEventCreate(&e0)); CK(cudaEventCreate(&e1));
  unsigned long long* d_bad; CK(cudaMalloc(&d_bad, 8));
  const int G = prop.multiProcessorCount * 4;
  int peer = (g_rank + 1) % g_world;
  std::vector<std::string> msgs; std::vector<int> fds;

  // ---------- B. legacy IPC ----------
  {
    float* buf; CK(cudaMalloc(&buf, BYTES));
    fill_kernel<<<G, 512>>>(buf, NF, (float)(g_rank + 1)); CK(cudaDeviceSynchronize());
    cudaIpcMemHandle_t h; CK(cudaIpcGetMemHandle(&h, buf));
    if (allgather(&h, sizeof h, -1, msgs, fds)) return -1;
    cudaIpcMemHandle_t ph; memcpy(&ph, msgs[peer].data(), sizeof ph);
    float* pbuf = nullptr; cudaError_t e = cudaIpcOpenMemHandle((void**)&pbuf, ph, cudaIpcMemLazyEnablePeerAccess);
    if (e != cudaSuccess) { printf("[r%d] PROBE legacy_ipc open FAILED: %s\n", g_rank, cudaGetErrorString(e)); cudaGetLastError(); }
    else {
      CK(cudaMemset(d_bad, 0, 8));
      check_kernel<<<G, 512>>>(pbuf, NF, (float)(peer + 1), d_bad);
      unsigned long long bad = 1; e = cudaMemcpy(&bad, d_bad, 8, cudaMemcpyDeviceToHost);
      printf("[r%d] PROBE legacy_ipc read peer %d: %s bad=%llu\n", g_rank, peer, e == cudaSuccess ? "ok" : cudaGetErrorString(e), bad);
      // bandwidth pull / push
      uint4* tmp; CK(cudaMalloc(&tmp, BYTES));
      for (int mode = 0; mode < 2; mode++) {
        if (barrier()) return -1;
        for (int it = 0; it < 2; it++) { if (mode == 0) copy_kernel<8><<<G, 512>>>(tmp, (const uint4*)pbuf, BYTES / 16); else copy_kernel<8><<<G, 512>>>((uint4*)pbuf, tmp, BYTES / 16); }
        CK(cudaDeviceSynchronize()); if (barrier()) return -1;
        CK(cudaEventRecord(e0));
        for (int it = 0; it < 5; it++) { if (mode == 0) copy_kernel<8><<<G, 512>>>(tmp, (const uint4*)pbuf, BYTES / 16); else copy_kernel<8><<<G, 512>>>((uint4*)pbuf, tmp, BYTES / 16); }
        CK(cudaEventRecord(e1)); CK(cudaDeviceSynchronize());
        printf("[r%d] PROBE ipc %s peer BW (all ranks concurrently, ring): %.1f GB/s\n", g_rank, mode == 0 ? "PULL(ld)" : "PUSH(st)", 5.0 * BYTES / time_ms(e0, e1) / 1e6);
      }
      // local copy for reference
      { uint4* tmp2; CK(cudaMalloc(&tmp2, BYTES)); copy_kernel<8><<<G, 512>>>(tmp2, tmp, BYTES / 16); CK(cudaEventRecord(e0));
        for (int it = 0; it < 5; it++) copy_kernel<8><<<G, 512>>>(tmp2, tmp, BYTES / 16);
        CK(cudaEventRecord(e1)); CK(cudaDeviceSynchronize());
        if (g_rank == 0) printf("[r0] PROBE local copy kernel: %.1f GB/s (r+w)\n", 2 * 5.0 * BYTES / time_ms(e0, e1) / 1e6); cudaFree(tmp2); }
      // flag ping-pong rank0 <-> rank1
      if (g_world >= 2) {
        CK(cudaMemset(buf, 0, 4096)); CK(cudaDeviceSynchronize()); if (barrier()) return -1;
        if (g_rank < 2 && peer == (g_rank ^ 1) || (g_rank < 2 && g_world > 2)) {
          // need handle of rank^1 specifically
          float* fb = pbuf;
          if (peer != (g_rank ^ 1)) { cudaIpcMemHandle_t h2; memcpy(&h2, msgs[g_rank ^ 1].data(), sizeof h2); CK(cudaIpcOpenMemHandle((void**)&fb, h2, cudaIpcMemLazyEnablePeerAccess)); }
          long long* d_cyc; CK(cudaMalloc(&d_cyc, 8));
          CK(cudaEventRecord(e0));
          pingpong_kernel<<<1, 1>>>((volatile unsigned*)buf, (unsigned*)fb, 1000, g_rank == 0, d_cyc);
          CK(cudaEventRecord(e1)); CK(cudaDeviceSynchronize());
          printf("[r%d] PROBE flag ping-pong: %.2f us per round trip (1000 iters)\n", g_rank, time_ms(e0, e1) * 1e3 / 1000);
        }
        if (barrier()) return -1;
      }
      cudaFree(tmp);
    }
    fflush(stdout);
  }

  // ---------- C. VMM + posix fd ----------
  Vmm mine = {}; std::vector<Vmm> peers(g_world);
  size_t gran = 0; bool vmm_ok = false;
  {
    CUmemAllocationProp ap = {}; ap.type = CU_MEM_ALLOCATION_TYPE_PINNED; ap.location.type = CU_MEM_LOCATION_TYPE_DEVICE; ap.location.id = cudev;
    ap.requestedHandleTypes = CU_MEM_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR;
    size_t gmin = 0, grec = 0;
    CU(cuMemGetAllocationGranularity(&gmin, &ap, CU_MEM_ALLOC_GRANULARITY_MINIMUM));
    CU(cuMemGetAllocationGranularity(&grec, &ap, CU_MEM_ALLOC_GRANULARITY_RECOMMENDED));
    size_t mcg = 0;
    if (a_mc) { CUmulticastObjectProp mp = {}; mp.numDevices = g_world; mp.size = BYTES; mp.handleTypes = CU_MEM_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR;
      CUresult r = cuMulticastGetGranularity(&mcg, &mp, CU_MULTICAST_GRANULARITY_RECOMMENDED); if (r != CUDA_SUCCESS) mcg = 0; }
    gran = grec > mcg ? grec : mcg;
    if (g_rank == 0) printf("PROBE vmm granularity min=%zu rec=%zu mc_rec=%zu\n", gmin, grec, mcg);
    mine.size = (BYTES + gran - 1) / gran * gran;
    CU(cuMemCreate(&mine.h, mine.size, &ap, 0));
    CU(cuMemAddressReserve(&mine.va, mine.size, gran, 0, 0));
    CU(cuMemMap(mine.va, mine.size, 0, mine.h, 0));
    CUmemAccessDesc ad = {}; ad.location.type = CU_MEM_LOCATION_TYPE_DEVICE; ad.location.id = cudev; ad.flags = CU_MEM_ACCESS_FLAGS_PROT_READWRITE;
    CU(cuMemSetAccess(mine.va, mine.size, &ad, 1));
    fill_kernel<<<G, 512>>>((float*)mine.va, NF, (float)(g_rank + 1)); CK(cudaDeviceSynchronize());
    int fd = -1; CUresult r = cuMemExportToShareableHandle(&fd, mine.h, CU_MEM_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR, 0);
    if (r != CUDA_SUCCESS) { printf("[r%d] PROBE vmm export FAILED %d\n", g_rank, (int)r); fd = -1; }
    char c = 0; if (allgather(&c, 1, fd, msgs, fds)) return -1;
    vmm_ok = true;
    for (int j = 0; j < g_world; j++) {
      if (j == g_rank) { peers[j] = mine; continue; }
      if (fds[j] < 0) { vmm_ok = false; continue; }
      Vmm p = {}; p.size = mine.size;
      r = cuMemImportFromShareableHandle(&p.h, (void*)(uintptr_t)fds[j], CU_MEM_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR);
      if (r != CUDA_SUCCESS) { printf("[r%d] PROBE vmm import from %d FAILED %d\n", g_rank, j, (int)r); vmm_ok = false; continue; }
      CU(cuMemAddressReserve(&p.va, p.size, gran, 0, 0));
      r = cuMemMap(p.va, p.size, 0, p.h, 0); if (r != CUDA_SUCCESS) { printf("[r%d] PROBE vmm map peer %d FAILED %d\n", g_rank, j, (int)r); vmm_ok = false; continue; }
      r = cuMemSetAccess(p.va, p.size, &ad, 1); if (r != CUDA_SUCCESS) { printf("[r%d] PROBE vmm setaccess peer %d FAILED %d\n", g_rank, j, (int)r); vmm_ok = false; continue; }
      peers[j] = p; close(fds[j]);
    }
    if (vmm_ok) {
      CK(cudaMemset(d_bad, 0, 8));
      check_kernel<<<G, 512>>>((const float*)peers[peer].va, NF, (float)(peer + 1), d_bad);
      unsigned long long bad = 1; cudaError_t e = cudaMemcpy(&bad, d_bad, 8, cudaMemcpyDeviceToHost);
      printf("[r%d] PROBE vmm read peer %d: %s bad=%llu\n", g_rank, peer, e == cudaSuccess ? "ok" : cudaGetErrorString(e), bad);
      uint4* tmp; CK(cudaMalloc(&tmp, BYTES));
      if (barrier()) return -1;
      copy_kernel<8><<<G, 512>>>(tmp, (const uint4*)peers[peer].va, BYTES / 16);
      CK(cudaDeviceSynchronize()); if (barrier()) return -1;
      CK(cudaEventRecord(e0)); for (int it = 0; it < 5; it++) copy_kernel<8><<<G, 512>>>(tmp, (const uint4*)peers[peer].va, BYTES / 16);
      CK(cudaEventRecord(e1)); CK(cudaDeviceSynchronize());
      printf("[r%d] PROBE vmm PULL ring BW: %.1f GB/s\n", g_rank, 5.0 * BYTES / time_ms(e0, e1) / 1e6);
      // grid-size sensitivity for pull
      for (int mult = 1; mult <= 8; mult *= 2) {
        int g2 = prop.multiProcessorCount * mult; if (barrier()) return -1;
        CK(cudaEventRecord(e0)); for (int it = 0; it < 3; it++) copy_kernel<8><<<g2, 512>>>(tmp, (const uint4*)peers[peer].va, BYTES / 16);
        CK(cudaEventRecord(e1)); CK(cudaDeviceSynchronize());
        if (g_rank == 0) printf("[r0] PROBE vmm PULL grid=%dxSMs: %.1f GB/s\n", mult, 3.0 * BYTES / time_ms(e0, e1) / 1e6);
      }
      // all-peer pull (two-shot pattern): slice s from rank s
      Ptrs ps; for (int j = 0; j < g_world; j++) ps.p[j] = (const uint4*)peers[j].va;
      if (barrier()) return -1;
      multi_pull_kernel<8><<<G, 512>>>(tmp, ps, g_world, BYTES / 16 / g_world); CK(cudaDeviceSynchronize()); if (barrier()) return -1;
      CK(cudaEventRecord(e0)); for (int it = 0; it < 5; it++) multi_pull_kernel<8><<<G, 512>>>(tmp, ps, g_world, BYTES / 16 / g_world);
      CK(cudaEventRecord(e1)); CK(cudaDeviceSynchronize());
      printf("[r%d] PROBE vmm ALL-PEER PULL (1/W from each incl self): total %.1f GB/s, remote part %.1f GB/s\n", g_rank,
             5.0 * BYTES / time_ms(e0, e1) / 1e6, 5.0 * BYTES * (g_world - 1) / g_world / time_ms(e0, e1) / 1e6);
      cudaFree(tmp);
    }
    fflush(stdout);
  }

  // ---------- D. multicast ----------
  if (a_mc && vmm_ok) {
    CUmemGenericAllocationHandle mch = 0; int mfd = -1;
    CUmulticastObjectProp mp = {}; mp.numDevices = g_world; mp.size = mine.size; mp.handleTypes = CU_MEM_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR;
    if (g_rank == 0) {
      CUresult r = cuMulticastCreate(&mch, &mp);
      if (r != CUDA_SUCCESS) { printf("[r0] PROBE cuMulticastCreate FAILED %d\n", (int)r); }
      else { r = cuMemExportToShareableHandle(&mfd, mch, CU_MEM_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR, 0); if (r != CUDA_SUCCESS) { printf("[r0] PROBE mc export FAILED %d\n", (int)r); mfd = -1; } }
    }
    char c = 0; if (allgather(&c, 1, g_rank == 0 ? mfd : -1, msgs, fds)) return -1;
    bool ok = true;
    if (g_rank != 0) {
      if (fds[0] < 0) ok = false;
      else { CUresult r = cuMemImportFromShareableHandle(&mch, (void*)(uintptr_t)fds[0], CU_MEM_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR); if (r != CUDA_SUCCESS) { printf("[r%d] PROBE mc import FAILED %d\n", g_rank, (int)r); ok = false; } }
    } else ok = (mfd >= 0);
    if (ok) { CUresult r = cuMulticastAddDevice(mch, cudev); if (r != CUDA_SUCCESS) { printf("[r%d] PROBE cuMulticastAddDevice FAILED %d\n", g_rank, (int)r); ok = false; } }
    if (barrier()) return -1;
    if (ok) { CUresult r = cuMulticastBindMem(mch, 0, mine.h, 0, mine.size, 0); if (r != CUDA_SUCCESS) { printf("[r%d] PROBE cuMulticastBindMem FAILED %d\n", g_rank, (int)r); ok = false; } }
    if (barrier()) return -1;
    CUdeviceptr mcva = 0;
    if (ok) {
      CU(cuMemAddressReserve(&mcva, mine.size, gran, 0, 0));
      CUresult r = cuMemMap(mcva, mine.size, 0, mch, 0); if (r != CUDA_SUCCESS) { printf("[r%d] PROBE mc map FAILED %d\n", g_rank, (int)r); ok = false; }
      CUmemAccessDesc ad = {}; ad.location.type = CU_MEM_LOCATION_TYPE_DEVICE; ad.location.id = cudev; ad.flags = CU_MEM_ACCESS_FLAGS_PROT_READWRITE;
      if (ok) { r = cuMemSetAccess(mcva, mine.size, &ad, 1); if (r != CUDA_SUCCESS) { printf("[r%d] PROBE mc setaccess FAILED %d\n", g_rank, (int)r); ok = false; } }
    }
    char okc = ok; if (allgather(&okc, 1, -1, msgs, fds)) return -1;
    for (int j = 0; j < g_world; j++) ok = ok && msgs[j][0];
    if (ok) {
      float* tmp; CK(cudaMalloc(&tmp, BYTES));
      fill_kernel<<<G, 512>>>((float*)mine.va, NF, (float)(g_rank + 1)); CK(cudaDeviceSynchronize()); if (barrier()) return -1;
      mc_ldreduce_kernel<<<G, 512>>>((float4*)tmp, (const float4*)mcva, BYTES / 16);
      CK(cudaMemset(d_bad, 0, 8)); check_kernel<<<G, 512>>>(tmp, NF, (float)(g_world * (g_world + 1) / 2), d_bad);
      unsigned long long bad = 1; cudaError_t e = cudaMemcpy(&bad, d_bad, 8, cudaMemcpyDeviceToHost);
      printf("[r%d] PROBE multimem.ld_reduce f32: %s bad=%llu\n", g_rank, e == cudaSuccess ? "ok" : cudaGetErrorString(e), bad);
      if (barrier()) return -1;
      CK(cudaEventRecord(e0)); for (int it = 0; it < 5; it++) mc_ldreduce_kernel<<<G, 512>>>((float4*)tmp, (const float4*)mcva, BYTES / 16);
      CK(cudaEventRecord(e1)); CK(cudaDeviceSynchronize());
      printf("[r%d] PROBE multimem.ld_reduce f32 full-buffer on all ranks: %.1f GB/s out\n", g_rank, 5.0 * BYTES / time_ms(e0, e1) / 1e6);
      if (barrier()) return -1;
      CK(cudaEventRecord(e0)); for (int it = 0; it < 5; it++) mc_ldreduce_bf16_kernel<<<G, 512>>>((uint4*)tmp, (const uint4*)mcva, BYTES / 16);
      CK(cudaEventRecord(e1)); CK(cudaDeviceSynchronize());
      printf("[r%d] PROBE multimem.ld_reduce bf16x2 full-buffer: %.1f GB/s out\n", g_rank, 5.0 * BYTES / time_ms(e0, e1) / 1e6);
      // sliced ld_reduce (each rank its 1/W slice) = reduce-scatter phase
      size_t sl16 = BYTES / 16 / g_world; if (barrier()) return -1;
      CK(cudaEventRecord(e0)); for (int it = 0; it < 5; it++) mc_ldreduce_kernel<<<G, 512>>>((float4*)tmp, (const float4*)mcva + g_rank * sl16, sl16);
      CK(cudaEventRecord(e1)); CK(cudaDeviceSynchronize());
      printf("[r%d] PROBE multimem RS phase (1/W slice each): algBW(S/t) %.1f GB/s\n", g_rank, 5.0 * BYTES / time_ms(e0, e1) / 1e6);
      // multimem.st: each rank writes its slice
      fill_kernel<<<G, 512>>>(tmp, NF, 100.0f + g_rank); CK(cudaDeviceSynchronize()); if (barrier()) return -1;
      mc_st_kernel<<<G, 512>>>((float4*)mcva + g_rank * sl16, (const float4*)tmp, sl16); CK(cudaDeviceSynchronize()); if (barrier()) return -1;
      bad = 0; for (int j = 0; j < g_world; j++) { CK(cudaMemset(d_bad, 0, 8)); check_kernel<<<G, 512>>>((const float*)mine.va + j * sl16 * 4, sl16 * 4, 100.0f + j, d_bad); unsigned long long b = 1; CK(cudaMemcpy(&b, d_bad, 8, cudaMemcpyDeviceToHost)); bad += b; }
      printf("[r%d] PROBE multimem.st broadcast: bad=%llu\n", g_rank, bad);
      if (barrier()) return -1;
      CK(cudaEventRecord(e0)); for (int it = 0; it < 5; it++) mc_st_kernel<<<G, 512>>>((float4*)mcva + g_rank * sl16, (const float4*)tmp, sl16);
      CK(cudaEventRecord(e1)); CK(cudaDeviceSynchronize());
      printf("[r%d] PROBE multimem AG phase (1/W slice each): algBW(S/t) %.1f GB/s\n", g_rank, 5.0 * BYTES / time_ms(e0, e1) / 1e6);
      if (barrier()) return -1;
      for (int mult = 1; mult <= 8; mult *= 2) {
        int g2 = prop.multiProcessorCount * mult; if (barrier()) return -1;
        CK(cudaEventRecord(e0)); for (int it = 0; it < 5; it++) mc_allreduce_kernel<<<g2, 512>>>((float4*)mcva, g_rank * sl16, sl16);
        CK(cudaEventRecord(e1)); CK(cudaDeviceSynchronize());
        printf("[r%d] PROBE multimem fused RS+AG (no sync) grid=%dxSMs: algBW %.1f GB/s busBW %.1f GB/s\n", g_rank, mult, 5.0 * BYTES / time_ms(e0, e1) / 1e6,
               5.0 * BYTES / time_ms(e0, e1) / 1e6 * 2 * (g_world - 1) / g_world);
      }
      if (g_exp) {
        // ---- E1: how many CTAs does NVLS need? (fused ld_reduce+st of the own 1/W slice)
        for (int g2 : {8, 16, 32, 64, 132, 264}) {
          if (barrier()) return -1;
          CK(cudaEventRecord(e0)); for (int it = 0; it < 5; it++) mc_allreduce_kernel<<<g2, 512>>>((float4*)mcva, g_rank * sl16, sl16);
          CK(cudaEventRecord(e1)); CK(cudaDeviceSynchronize());
          if (g_rank == 0) printf("[r0] EXP E1 nvls grid=%d CTAs: algBW %.1f GB/s\n", g2, 5.0 * BYTES / time_ms(e0, e1) / 1e6);
        }
        // ---- E5: one source: rank 0 alone multicasts the whole buffer
        if (barrier()) return -1;
        CK(cudaEventRecord(e0));
        if (g_rank == 0) for (int it = 0; it < 5; it++) mc_st_kernel<<<G, 512>>>((float4*)mcva, (const float4*)tmp, BYTES / 16);
        CK(cudaEventRecord(e1)); CK(cudaDeviceSynchronize());
        if (g_rank == 0) printf("[r0] EXP E5 single-source multimem.st: %.1f GB/s out of the root\n", 5.0 * BYTES / time_ms(e0, e1) / 1e6);
        // ---- E2: does unicast P2P traffic ride beside NVLS?  first half of the buffer: NVLS; second half: P2P landing zone
        if (g_world > 2) {
          Ptrs ps; for (int j = 0; j < g_world; j++) ps.p[j] = (const uint4*)peers[j].va;
          size_t half16 = BYTES / 32, nsl16 = half16 / g_world;      // NVLS slice per rank inside the first half
          size_t p2p16 = half16 / g_world / (g_world - 1) * (g_world - 1);  // bytes each rank pushes in total (lands in 1/W of the peers' second half)
          struct { int n_nvls, n_p2p; size_t nv, np; const char* name; } cfg[] = {
              {32, 0, nsl16, 0, "NVLS only (32 CTAs)"}, {0, 264, 0, p2p16, "P2P only (264 CTAs)"}, {32, 264, nsl16, p2p16, "both"}};
          for (auto& c : cfg) {
            if (barrier()) return -1;
            CK(cudaEventRecord(e0));
            for (int it = 0; it < 5; it++)
              mix_kernel<<<c.n_nvls + c.n_p2p, 512>>>((float4*)mcva, g_rank * nsl16, c.nv, c.n_nvls, ps, g_rank, g_world, (const uint4*)tmp, half16, c.np);
            CK(cudaEventRecord(e1)); CK(cudaDeviceSynchronize());
            double ms = time_ms(e0, e1) / 5;
            if (g_rank == 0) printf("[r0] EXP E2 %-22s %.1f us  (NVLS algBW %.1f GB/s over %zu MB; P2P egress %.1f GB/s)\n", c.name, ms * 1e3,
                                    c.nv ? half16 * 16.0 / ms / 1e6 : 0.0, half16 * 16 >> 20, c.np ? c.np * 16.0 / ms / 1e6 : 0.0);
          }
        }
        // ---- E3: fence cost with and without a concurrent store stream to the peer (one CTA per SM)
        {
          long long* d_cyc; CK(cudaMalloc(&d_cyc, 8));
          unsigned* pflag = (unsigned*)((char*)peers[peer].va + (BYTES / 2));   // scratch words inside the landing zone
          for (int stream = 0; stream < 2; stream++) {
            if (barrier()) return -1;
            fence_kernel<<<prop.multiProcessorCount, 512>>>((uint4*)peers[peer].va + BYTES / 32 + 4096, (const uint4*)tmp, (BYTES / 64), pflag, 200, stream, d_cyc);
            long long cyc = 0; CK(cudaMemcpy(&cyc, d_cyc, 8, cudaMemcpyDeviceToHost));
            if (g_rank == 0) printf("[r0] EXP E3 fence.acq_rel.sys + flag store, %s: %lld cycles each (%.2f us at %.0f MHz)\n",
                                    stream ? "other warps streaming stores to the peer" : "quiet SM", cyc, cyc / (prop.clockRate / 1e3), prop.clockRate / 1e3);
          }
          cudaFree(d_cyc);
        }
        // ---- E4: packed data+flag round trip (no fence) between rank 0 and 1
        if (g_world >= 2) {
          CK(cudaMemset((void*)mine.va, 0, 4096)); CK(cudaDeviceSynchronize()); if (barrier()) return -1;
          if (g_rank < 2) {
            CK(cudaEventRecord(e0));
            ll_pingpong_kernel<<<1, 1>>>((uint4*)mine.va, (uint4*)peers[g_rank ^ 1].va, 1000, g_rank == 0);
            CK(cudaEventRecord(e1)); CK(cudaDeviceSynchronize());
            printf("[r%d] EXP E4 packed 16-byte data+flag ping-pong: %.2f us per round trip\n", g_rank, time_ms(e0, e1));
          }
          if (barrier()) return -1;
        }
      }
      cudaFree(tmp);
    } else printf("[r%d] PROBE multicast path NOT usable\n", g_rank);
    fflush(stdout);
  } else if (g_rank == 0) printf("PROBE multicast skipped (mc=%d vmm_ok=%d)\n", a_mc, (int)vmm_ok);
  if (barrier()) return -1;
  printf("[r%d] PROBE done\n", g_rank); fflush(stdout);
  return 0;
}

int main(int argc, char** argv) {
  int W = argc > 1 ? atoi(argv[1]) : 2; int isolate = argc > 2 && !strcmp(argv[2], "isolate");
  g_exp = argc > 2 && !strcmp(argv[2], "exp");
  std::vector<int> socks(W); std::vector<pid_t> pids(W);
  for (int r = 0; r < W; r++) {
    int sv[2]; if (socketpair(AF_UNIX, SOCK_STREAM, 0, sv)) { perror("socketpair"); return 1; }
    pid_t p = fork();
    if (p == 0) { close(sv[0]); for (int k = 0; k < r; k++) close(socks[k]); g_rank = r; g_world = W; g_sock = sv[1]; alarm(240); int rc = child_main(isolate); fflush(stdout); _exit(rc ? 1 : 0); }
    close(sv[1]); socks[r] = sv[0]; pids[r] = p;
  }
  // relay loop: rounds of allgather until a child closes
  alarm(300);
  for (;;) {
    std::vector<std::string> m(W); std::vector<int> f(W, -1); bool dead = false;
    for (int r = 0; r < W; r++) if (recv_msg(socks[r], m[r], &f[r])) { dead = true; break; }
    if (dead) break;
    for (int r = 0; r < W; r++) for (int j = 0; j < W; j++) send_msg(socks[r], m[j].data(), m[j].size(), f[j]);
    for (int j = 0; j < W; j++) if (f[j] >= 0) close(f[j]);
  }
  int rc = 0; for (int r = 0; r < W; r++) { int st; waitpid(pids[r], &st, 0); if (!WIFEXITED(st) || WEXITSTATUS(st)) rc = 1; }
  printf("PROBE exit rc=%d\n", rc);
  return rc;
}
