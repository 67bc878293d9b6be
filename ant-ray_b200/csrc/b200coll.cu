// Host side of the C-ABI declared in include/b200coll.h: arena creation and sharing (VMM + POSIX fd,
// or legacy CUDA IPC), NVSwitch multicast binding, algorithm selection and kernel launches.
//
// The driver API (cuMem*, cuMulticast*) is reached through cudaGetDriverEntryPoint so the library
// has no link-time dependency on libcuda and can be loaded (symbol check) on a machine without a GPU.
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdarg.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <unistd.h>

#include <atomic>
#include <initializer_list>
#include <mutex>

#include "byte_kernels.cuh"
#include "launch_typed.cuh"
#include "norm_launch.h"
#include "se_launch.h"

using namespace b200c;

// ------------------------------------------------------------------------------------------------
// errors
// ------------------------------------------------------------------------------------------------
static thread_local char g_err[512] = "";
static int fail(int code, const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof g_err, fmt, ap);
  va_end(ap);
  return code;
}
#define RT(x)                                                                                      \
  do {                                                                                             \
    cudaError_t e_ = (x);                                                                          \
    if (e_ != cudaSuccess) return fail(B200C_ECUDA, "%s failed: %s", #x, cudaGetErrorString(e_)); \
  } while (0)

static std::atomic<uint64_t> g_launches{0};

// ------------------------------------------------------------------------------------------------
// driver entry points
// ------------------------------------------------------------------------------------------------
struct Driver {
  bool ok = false;
  CUresult (*GetErrorString)(CUresult, const char**) = nullptr;
  CUresult (*DeviceGet)(CUdevice*, int) = nullptr;
  CUresult (*DeviceGetAttribute)(int*, CUdevice_attribute, CUdevice) = nullptr;
  CUresult (*MemGetAllocationGranularity)(size_t*, const CUmemAllocationProp*, CUmemAllocationGranularity_flags) = nullptr;
  CUresult (*MemCreate)(CUmemGenericAllocationHandle*, size_t, const CUmemAllocationProp*, unsigned long long) = nullptr;
  CUresult (*MemRelease)(CUmemGenericAllocationHandle) = nullptr;
  CUresult (*MemAddressReserve)(CUdeviceptr*, size_t, size_t, CUdeviceptr, unsigned long long) = nullptr;
  CUresult (*MemAddressFree)(CUdeviceptr, size_t) = nullptr;
  CUresult (*MemMap)(CUdeviceptr, size_t, size_t, CUmemGenericAllocationHandle, unsigned long long) = nullptr;
  CUresult (*MemUnmap)(CUdeviceptr, size_t) = nullptr;
  CUresult (*MemSetAccess)(CUdeviceptr, size_t, const CUmemAccessDesc*, size_t) = nullptr;
  CUresult (*MemExportToShareableHandle)(void*, CUmemGenericAllocationHandle, CUmemAllocationHandleType, unsigned long long) = nullptr;
  CUresult (*MemImportFromShareableHandle)(CUmemGenericAllocationHandle*, void*, CUmemAllocationHandleType) = nullptr;
  CUresult (*MulticastCreate)(CUmemGenericAllocationHandle*, const CUmulticastObjectProp*) = nullptr;
  CUresult (*MulticastAddDevice)(CUmemGenericAllocationHandle, CUdevice) = nullptr;
  CUresult (*MulticastBindMem)(CUmemGenericAllocationHandle, size_t, CUmemGenericAllocationHandle, size_t, size_t, unsigned long long) = nullptr;
  CUresult (*MulticastUnbind)(CUmemGenericAllocationHandle, CUdevice, size_t, size_t) = nullptr;
  CUresult (*MulticastGetGranularity)(size_t*, const CUmulticastObjectProp*, CUmulticastGranularity_flags) = nullptr;
};
static Driver g_drv;
static std::once_flag g_drv_once;

template <typename F>
static bool load_sym(const char* name, F* out) {
  void* p = nullptr;
  cudaDriverEntryPointQueryResult q;
  if (cudaGetDriverEntryPoint(name, &p, cudaEnableDefault, &q) != cudaSuccess || q != cudaDriverEntryPointSuccess || !p) {
    cudaGetLastError();
    return false;
  }
  *out = reinterpret_cast<F>(p);
  return true;
}
static void load_driver() {
  Driver& d = g_drv;
  bool ok = true;
  ok &= load_sym("cuGetErrorString", &d.GetErrorString);
  ok &= load_sym("cuDeviceGet", &d.DeviceGet);
  ok &= load_sym("cuDeviceGetAttribute", &d.DeviceGetAttribute);
  ok &= load_sym("cuMemGetAllocationGranularity", &d.MemGetAllocationGranularity);
  ok &= load_sym("cuMemCreate", &d.MemCreate);
  ok &= load_sym("cuMemRelease", &d.MemRelease);
  ok &= load_sym("cuMemAddressReserve", &d.MemAddressReserve);
  ok &= load_sym("cuMemAddressFree", &d.MemAddressFree);
  ok &= load_sym("cuMemMap", &d.MemMap);
  ok &= load_sym("cuMemUnmap", &d.MemUnmap);
  ok &= load_sym("cuMemSetAccess", &d.MemSetAccess);
  ok &= load_sym("cuMemExportToShareableHandle", &d.MemExportToShareableHandle);
  ok &= load_sym("cuMemImportFromShareableHandle", &d.MemImportFromShareableHandle);
  // multicast is optional
  load_sym("cuMulticastCreate", &d.MulticastCreate);
  load_sym("cuMulticastAddDevice", &d.MulticastAddDevice);
  load_sym("cuMulticastBindMem", &d.MulticastBindMem);
  load_sym("cuMulticastUnbind", &d.MulticastUnbind);
  load_sym("cuMulticastGetGranularity", &d.MulticastGetGranularity);
  d.ok = ok;
}
static const char* cu_str(CUresult r) {
  const char* s = nullptr;
  if (g_drv.GetErrorString) g_drv.GetErrorString(r, &s);
  return s ? s : "unknown";
}
#define DRV(call)                                                                                   \
  do {                                                                                              \
    CUresult r_ = (call);                                                                           \
    if (r_ != CUDA_SUCCESS) return fail(B200C_ECUDA, "%s failed: %d (%s)", #call, (int)r_, cu_str(r_)); \
  } while (0)

struct DeviceGuard {
  int prev = -1, dev;
  bool switched = false;
  explicit DeviceGuard(int d) : dev(d) {
    if (cudaGetDevice(&prev) == cudaSuccess && prev != d) { cudaSetDevice(d); switched = true; }
  }
  ~DeviceGuard() { if (switched) cudaSetDevice(prev); }
};

// ------------------------------------------------------------------------------------------------
// communicator
// ------------------------------------------------------------------------------------------------
struct b200c_comm {
  int rank = 0, world = 1, device = 0;
  CUdevice cudev = 0;
  b200c_config_t cfg{};
  int sm_count = 132;
  // arena
  size_t arena_bytes = 0, gran = 0;
  size_t off_staging = 0, off_p2p = 0, off_mring = 0, off_ll = 0, ll_words = 0, off_sym = 0, sym_bytes = 0;
  uint32_t mcells = 0;
  uint64_t layout_hash = 0;
  bool vmm = true;
  CUmemGenericAllocationHandle own_handle = 0;
  CUmemGenericAllocationHandle peer_handle[kMaxRanks] = {};
  char* arena[kMaxRanks] = {};
  bool imported[kMaxRanks] = {};
  // multicast
  CUmemGenericAllocationHandle mc_handle = 0;
  bool mc_have_handle = false, mc_added = false, mc_bound = false;
  char* mc_arena = nullptr;
  // status
  Status* status_host = nullptr;
  Status* status_dev = nullptr;
  // state
  bool ready = false, destroyed = false;
  uint32_t seq = 0;
  bool bcast_mc = false;   // broadcast through one multicast store stream (wins for W > 2)
  uint32_t pipe_base = 0;  // flag epoch of the round-pipelined kernels (advanced by the round count of each op)
  uint32_t ll_seq = 0;     // LL op counter (flag value of the packed stores; region half = ll_seq & 1)
  int local_scale_ctas_per_sm = 0, tma_ctas_per_sm = 0;
  // multi-stream NVLS pipeline: internal streams (copy-in, switch, copy-out) and per-region events
  cudaStream_t ps_in = nullptr, ps_nv = nullptr, ps_out = nullptr;
  cudaEvent_t pe_start = nullptr, pe_in[8] = {}, pe_nv[8] = {}, pe_out[8] = {};
  uint32_t send_cells[kMaxRanks] = {};
  uint32_t recv_cells[kMaxRanks] = {};
  uint32_t msend_cells = 0;            // multi-reader ring of this rank: cells sent so far
  uint32_t msend_mask = 0;             // ... and its (fixed) reader set, 0 = not chosen yet
  uint32_t mrecv_cells[kMaxRanks] = {};
  DevComm dev{};
};

static size_t round_up(size_t x, size_t a) { return (x + a - 1) / a * a; }
static int load_kernels(int device);

// symmetric pool state (see b200c_pool_bind)
struct PoolBlock { size_t off, len; };
static std::mutex g_pool_mu;
static b200c_comm* g_pool_comm = nullptr;
static PoolBlock g_pool_free[4096];
static int g_pool_nfree = 0;
constexpr size_t kPoolGran = 2ull << 20;


extern "C" int b200c_version(void) { return B200C_VERSION; }
extern "C" const char* b200c_last_error(void) { return g_err; }
extern "C" const char* b200c_status_string(int s) {
  switch (s) {
    case B200C_OK: return "ok";
    case B200C_EINVAL: return "invalid argument";
    case B200C_ECUDA: return "CUDA error";
    case B200C_ESTATE: return "communicator not ready or destroyed";
    case B200C_EUNSUPPORTED: return "unsupported dtype/op/algorithm";
    case B200C_ETIMEOUT: return "timed out waiting for a peer";
    case B200C_EABORTED: return "communicator aborted";
    case B200C_EMISMATCH: return "peers disagree on the collective's arguments";
    case B200C_ENOMEM: return "out of memory";
    default: return "unknown status";
  }
}
extern "C" size_t b200c_dtype_size(int dtype) {
  switch (dtype) {
    case B200C_INT8: case B200C_UINT8: return 1;
    case B200C_FLOAT16: case B200C_BFLOAT16: return 2;
    case B200C_INT32: case B200C_UINT32: case B200C_FLOAT32: return 4;
    case B200C_INT64: case B200C_UINT64: case B200C_FLOAT64: return 8;
    default: return 0;
  }
}
extern "C" uint64_t b200c_launch_count(void) { return g_launches.load(); }

extern "C" void b200c_default_config(b200c_config_t* cfg) {
  memset(cfg, 0, sizeof *cfg);
  cfg->struct_size = sizeof *cfg;
  cfg->share_mode = B200C_SHARE_VMM_FD;
  cfg->staging_bytes = 256ull << 20;
  cfg->symmetric_bytes = 0;
  cfg->p2p_slot_bytes = 32ull << 10;
  cfg->p2p_slots = 1024;   // 32 MiB per ordered pair: the ring must hold the data a ready/ack round trip is behind
  cfg->max_blocks = 264;   // 2 CTAs of 512 threads on each of the 132 SMs of an H100
  cfg->oneshot_max_bytes = 0;  // 0 = pick by world size in b200c_comm_create
  cfg->nvls_min_bytes = (1ull << 20) + 1;
  cfg->nvls_pipe_min_bytes = 32ull << 20;  // staged NVLS pieces from 32 MiB up run round-pipelined
  cfg->timeout_ms = 600000;  // a slow peer (data loading, first-step autotuning skew) is not a dead peer
  cfg->granule_bytes = 32ull << 10;
  cfg->ll_max_bytes = 64ull << 10;
  cfg->bcast_rounds_min_bytes = 4ull << 20;
  cfg->nvls_unroll = 4;
  cfg->nvls_streams_min_bytes = 768ull << 20;
  cfg->nvls_streams_piece_bytes = 128ull << 20;
  cfg->rounds_order = 0;
  cfg->nvls_lanes = 48;
  cfg->lane_granule_bytes = 64ull << 10;
  cfg->nvls_lanes_min_bytes = 0;   // opt-in until measured on the target box
  cfg->nvls_blocks = 32;   // zero-copy NVLS: a few CTAs saturate the switch; more only scatter the access pattern
}

static int ensure_driver() {
  std::call_once(g_drv_once, load_driver);
  if (!g_drv.ok) return fail(B200C_ECUDA, "CUDA driver entry points unavailable (no GPU driver?)");
  return B200C_OK;
}

extern "C" int b200c_device_props(int device, b200c_props_t* out) {
  if (!out) return fail(B200C_EINVAL, "out is null");
  memset(out, 0, sizeof *out);
  int n = 0;
  if (cudaGetDeviceCount(&n) != cudaSuccess || device < 0 || device >= n) {
    cudaGetLastError();
    return fail(B200C_ECUDA, "no CUDA device %d (count %d)", device, n);
  }
  int rc = ensure_driver();
  if (rc) return rc;
  cudaDeviceProp p;
  RT(cudaGetDeviceProperties(&p, device));
  out->device = device;
  out->sm_count = p.multiProcessorCount;
  out->cc_major = p.major;
  out->cc_minor = p.minor;
  out->total_mem = p.totalGlobalMem;
  DeviceGuard g(device);
  RT(cudaFree(0));
  CUdevice cd;
  DRV(g_drv.DeviceGet(&cd, device));
  g_drv.DeviceGetAttribute(&out->vmm_supported, CU_DEVICE_ATTRIBUTE_VIRTUAL_MEMORY_MANAGEMENT_SUPPORTED, cd);
  g_drv.DeviceGetAttribute(&out->posix_fd_supported, CU_DEVICE_ATTRIBUTE_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR_SUPPORTED, cd);
  g_drv.DeviceGetAttribute(&out->multicast_supported, CU_DEVICE_ATTRIBUTE_MULTICAST_SUPPORTED, cd);
  return B200C_OK;
}

static CUmemAllocationProp alloc_prop(CUdevice cd) {
  CUmemAllocationProp ap;
  memset(&ap, 0, sizeof ap);
  ap.type = CU_MEM_ALLOCATION_TYPE_PINNED;
  ap.location.type = CU_MEM_LOCATION_TYPE_DEVICE;
  ap.location.id = cd;
  ap.requestedHandleTypes = CU_MEM_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR;
  return ap;
}
static int map_handle(b200c_comm* c, CUmemGenericAllocationHandle h, char** out) {
  CUdeviceptr va = 0;
  DRV(g_drv.MemAddressReserve(&va, c->arena_bytes, c->gran, 0, 0));
  CUresult r = g_drv.MemMap(va, c->arena_bytes, 0, h, 0);
  if (r != CUDA_SUCCESS) { g_drv.MemAddressFree(va, c->arena_bytes); return fail(B200C_ECUDA, "cuMemMap failed: %d (%s)", (int)r, cu_str(r)); }
  CUmemAccessDesc ad;
  memset(&ad, 0, sizeof ad);
  ad.location.type = CU_MEM_LOCATION_TYPE_DEVICE;
  ad.location.id = c->cudev;
  ad.flags = CU_MEM_ACCESS_FLAGS_PROT_READWRITE;
  r = g_drv.MemSetAccess(va, c->arena_bytes, &ad, 1);
  if (r != CUDA_SUCCESS) { g_drv.MemUnmap(va, c->arena_bytes); g_drv.MemAddressFree(va, c->arena_bytes); return fail(B200C_ECUDA, "cuMemSetAccess failed: %d (%s)", (int)r, cu_str(r)); }
  *out = reinterpret_cast<char*>(va);
  return B200C_OK;
}

extern "C" int b200c_comm_create(int rank, int world, int device, const b200c_config_t* cfg_in, b200c_comm_t** out) {
  if (!out) return fail(B200C_EINVAL, "out is null");
  if (world < 1 || world > kMaxRanks) return fail(B200C_EINVAL, "world size %d not in [1, %d] (one NVSwitch domain)", world, kMaxRanks);
  if (rank < 0 || rank >= world) return fail(B200C_EINVAL, "rank %d not in [0, %d)", rank, world);
  int rc = ensure_driver();
  if (rc) return rc;
  b200c_config_t cfg;
  b200c_default_config(&cfg);
  if (cfg_in) {
    if (cfg_in->struct_size != sizeof(b200c_config_t)) return fail(B200C_EINVAL, "config struct_size %u != %zu", cfg_in->struct_size, sizeof(b200c_config_t));
    cfg = *cfg_in;
  }
  if (cfg.max_blocks == 0 || cfg.max_blocks > (uint32_t)kMaxBlocks) return fail(B200C_EINVAL, "max_blocks %u not in [1, %d]", cfg.max_blocks, kMaxBlocks);
  if (cfg.p2p_slots == 0 || cfg.p2p_slots > (uint32_t)kMaxCells) return fail(B200C_EINVAL, "p2p_slots %u not in [1, %d]", cfg.p2p_slots, kMaxCells);
  if (cfg.p2p_slot_bytes < 512 || cfg.p2p_slot_bytes % 16) return fail(B200C_EINVAL, "p2p_slot_bytes must be a multiple of 16 and >= 512");
  if (cfg.staging_bytes < (1u << 16) || cfg.staging_bytes % 4096) return fail(B200C_EINVAL, "staging_bytes must be a multiple of 4096 and >= 64 KiB");
  if (cfg.timeout_ms == 0) cfg.timeout_ms = 600000;
  if (cfg.granule_bytes == 0) cfg.granule_bytes = 32ull << 10;
  if (cfg.granule_bytes % 16384) return fail(B200C_EINVAL, "granule_bytes must be a multiple of 16 KiB");
  if (cfg.ll_max_bytes > (1ull << 20)) return fail(B200C_EINVAL, "ll_max_bytes must be <= 1 MiB");
  if (cfg.nvls_blocks > (uint32_t)kMaxBlocks) return fail(B200C_EINVAL, "nvls_blocks %u > %d", cfg.nvls_blocks, kMaxBlocks);
  if (cfg.nvls_lanes == 0) cfg.nvls_lanes = 48;
  if (cfg.nvls_lanes > cfg.max_blocks / 2) cfg.nvls_lanes = cfg.max_blocks / 2 ? cfg.max_blocks / 2 : 1;
  if (cfg.lane_granule_bytes == 0) cfg.lane_granule_bytes = 64ull << 10;
  if (cfg.lane_granule_bytes % 8192) return fail(B200C_EINVAL, "lane_granule_bytes must be a multiple of 8 KiB");
  if (cfg.nvls_streams_piece_bytes == 0) cfg.nvls_streams_piece_bytes = 128ull << 20;
  if (cfg.nvls_streams_piece_bytes % (1u << 20)) return fail(B200C_EINVAL, "nvls_streams_piece_bytes must be a multiple of 1 MiB");
  // one-shot (one flag round, (W-1)*S pushed) pays off for small messages, longer at W=2 where it moves the least
  if (cfg.oneshot_max_bytes == 0) cfg.oneshot_max_bytes = world <= 2 ? (8ull << 20) : (1ull << 20);

  int ndev = 0;
  RT(cudaGetDeviceCount(&ndev));
  if (device < 0 || device >= ndev) return fail(B200C_EINVAL, "device %d not visible (count %d)", device, ndev);
  DeviceGuard g(device);
  RT(cudaFree(0));
  rc = load_kernels(device);
  if (rc) return rc;
  b200c_comm* c = new b200c_comm();
  c->rank = rank; c->world = world; c->device = device; c->cfg = cfg;
  c->vmm = cfg.share_mode == B200C_SHARE_VMM_FD;
  cudaDeviceProp prop;
  RT(cudaGetDeviceProperties(&prop, device));
  c->sm_count = prop.multiProcessorCount;
  DRV(g_drv.DeviceGet(&c->cudev, device));

  // layout
  c->off_staging = kPadBytes;
  c->off_p2p = c->off_staging + 2 * cfg.staging_bytes;
  size_t p2p_bytes = world > 1 ? (size_t)world * cfg.p2p_slots * cfg.p2p_slot_bytes : 0;   // one ring per source rank
  c->mcells = world > 2 ? (cfg.p2p_slots < 64 ? cfg.p2p_slots : 64) : 0;  // with one possible reader the pairwise ring is the multi-reader ring
  c->off_mring = round_up(c->off_p2p + p2p_bytes, 4096);
  size_t mring_bytes = (size_t)world * c->mcells * cfg.p2p_slot_bytes;
  c->off_ll = round_up(c->off_mring + mring_bytes, 4096);
  c->ll_words = world > 1 ? round_up((cfg.ll_max_bytes + 3) / 4, 4) : 0;   // whole 16-byte vectors
  size_t ll_bytes = 2 * (size_t)kMaxRanks * c->ll_words * 8;
  c->off_sym = round_up(c->off_ll + ll_bytes, 2ull << 20);
  size_t want = c->off_sym + cfg.symmetric_bytes;
  size_t gran = 2ull << 20;
  if (c->vmm) {
    CUmemAllocationProp ap = alloc_prop(c->cudev);
    size_t g1 = 0;
    DRV(g_drv.MemGetAllocationGranularity(&g1, &ap, CU_MEM_ALLOC_GRANULARITY_RECOMMENDED));
    if (g1 > gran) gran = g1;
    int mc = 0;
    g_drv.DeviceGetAttribute(&mc, CU_DEVICE_ATTRIBUTE_MULTICAST_SUPPORTED, c->cudev);
    if (mc && g_drv.MulticastGetGranularity && world > 1) {
      CUmulticastObjectProp mp;
      memset(&mp, 0, sizeof mp);
      mp.numDevices = world; mp.size = round_up(want, gran); mp.handleTypes = CU_MEM_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR;
      size_t g2 = 0;
      if (g_drv.MulticastGetGranularity(&g2, &mp, CU_MULTICAST_GRANULARITY_MINIMUM) == CUDA_SUCCESS && g2 > gran) gran = g2;
    }
  }
  c->gran = gran;
  c->arena_bytes = round_up(want, gran);
  c->sym_bytes = c->arena_bytes - c->off_sym;
  c->layout_hash = (uint64_t)cfg.staging_bytes * 1000003ull ^ (uint64_t)cfg.p2p_slot_bytes * 10007ull ^ (uint64_t)cfg.p2p_slots * 101ull ^
                   (uint64_t)c->arena_bytes ^ ((uint64_t)cfg.max_blocks << 48) ^ ((uint64_t)world << 56) ^
                   (uint64_t)cfg.ll_max_bytes * 7919ull ^ (uint64_t)cfg.granule_bytes * 31ull ^ ((uint64_t)cfg.nvls_blocks << 36);

  if (c->vmm) {
    CUmemAllocationProp ap = alloc_prop(c->cudev);
    CUresult r = g_drv.MemCreate(&c->own_handle, c->arena_bytes, &ap, 0);
    if (r != CUDA_SUCCESS) { size_t ab = c->arena_bytes; delete c; return fail(r == CUDA_ERROR_OUT_OF_MEMORY ? B200C_ENOMEM : B200C_ECUDA, "cuMemCreate(%zu bytes) failed: %d (%s)", ab, (int)r, cu_str(r)); }
    rc = map_handle(c, c->own_handle, &c->arena[rank]);
    if (rc) { g_drv.MemRelease(c->own_handle); delete c; return rc; }
  } else {
    void* p = nullptr;
    cudaError_t e = cudaMalloc(&p, c->arena_bytes);
    if (e != cudaSuccess) { size_t ab = c->arena_bytes; delete c; return fail(e == cudaErrorMemoryAllocation ? B200C_ENOMEM : B200C_ECUDA, "cudaMalloc(%zu) failed: %s", ab, cudaGetErrorString(e)); }
    c->arena[rank] = static_cast<char*>(p);
  }
  c->imported[rank] = true;
  RT(cudaMemset(c->arena[rank], 0, kPadBytes));
  if (ll_bytes) RT(cudaMemset(c->arena[rank] + c->off_ll, 0, ll_bytes));  // LL flags start at 0 (never a valid ll_seq)
  RT(cudaHostAlloc(reinterpret_cast<void**>(&c->status_host), sizeof(Status), cudaHostAllocMapped | cudaHostAllocPortable));
  memset((void*)c->status_host, 0, sizeof(Status));
  RT(cudaHostGetDevicePointer(reinterpret_cast<void**>(&c->status_dev), (void*)c->status_host, 0));
  RT(cudaDeviceSynchronize());
  *out = c;
  return B200C_OK;
}

extern "C" int b200c_comm_export(b200c_comm_t* c, b200c_export_t* out) {
  if (!c || !out) return fail(B200C_EINVAL, "null argument");
  if (c->destroyed) return fail(B200C_ESTATE, "communicator destroyed");
  memset(out, 0, sizeof *out);
  out->share_mode = c->vmm ? B200C_SHARE_VMM_FD : B200C_SHARE_LEGACY_IPC;
  out->fd = -1;
  out->arena_bytes = c->arena_bytes;
  out->layout_hash = c->layout_hash;
  out->pid = (int32_t)getpid();
  DeviceGuard g(c->device);
  if (c->vmm) {
    int fd = -1;
    DRV(g_drv.MemExportToShareableHandle(&fd, c->own_handle, CU_MEM_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR, 0));
    out->fd = fd;
  } else {
    cudaIpcMemHandle_t h;
    RT(cudaIpcGetMemHandle(&h, c->arena[c->rank]));
    static_assert(sizeof h == 64, "cudaIpcMemHandle_t is 64 bytes");
    memcpy(out->ipc, &h, 64);
  }
  return B200C_OK;
}

extern "C" int b200c_comm_import(b200c_comm_t* c, int peer, const b200c_export_t* e) {
  if (!c || !e) return fail(B200C_EINVAL, "null argument");
  if (c->destroyed) return fail(B200C_ESTATE, "communicator destroyed");
  if (peer < 0 || peer >= c->world || peer == c->rank) return fail(B200C_EINVAL, "bad peer %d", peer);
  if (c->imported[peer]) return fail(B200C_ESTATE, "peer %d already imported", peer);
  if (e->arena_bytes != c->arena_bytes || e->layout_hash != c->layout_hash)
    return fail(B200C_EMISMATCH, "peer %d arena layout differs (bytes %llu vs %zu): all ranks must use the same config", peer,
                (unsigned long long)e->arena_bytes, c->arena_bytes);
  if ((e->share_mode == B200C_SHARE_VMM_FD) != c->vmm) return fail(B200C_EMISMATCH, "peer %d uses a different share mode", peer);
  DeviceGuard g(c->device);
  if (c->vmm) {
    if (e->fd < 0) return fail(B200C_EINVAL, "peer %d export carries no fd", peer);
    DRV(g_drv.MemImportFromShareableHandle(&c->peer_handle[peer], (void*)(uintptr_t)e->fd, CU_MEM_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR));
    int rc = map_handle(c, c->peer_handle[peer], &c->arena[peer]);
    if (rc) return rc;
  } else {
    cudaIpcMemHandle_t h;
    memcpy(&h, e->ipc, 64);
    void* p = nullptr;
    RT(cudaIpcOpenMemHandle(&p, h, cudaIpcMemLazyEnablePeerAccess));
    c->arena[peer] = static_cast<char*>(p);
  }
  c->imported[peer] = true;
  return B200C_OK;
}

extern "C" int b200c_comm_mc_create(b200c_comm_t* c, int* fd_out) {
  if (!c || !fd_out) return fail(B200C_EINVAL, "null argument");
  if (!c->vmm) return fail(B200C_EUNSUPPORTED, "multicast needs the VMM share mode");
  if (!g_drv.MulticastCreate) return fail(B200C_EUNSUPPORTED, "driver has no cuMulticastCreate");
  int mc = 0;
  g_drv.DeviceGetAttribute(&mc, CU_DEVICE_ATTRIBUTE_MULTICAST_SUPPORTED, c->cudev);
  if (!mc) return fail(B200C_EUNSUPPORTED, "device does not support multicast");
  DeviceGuard g(c->device);
  CUmulticastObjectProp mp;
  memset(&mp, 0, sizeof mp);
  mp.numDevices = c->world; mp.size = c->arena_bytes; mp.handleTypes = CU_MEM_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR;
  DRV(g_drv.MulticastCreate(&c->mc_handle, &mp));
  c->mc_have_handle = true;
  int fd = -1;
  DRV(g_drv.MemExportToShareableHandle(&fd, c->mc_handle, CU_MEM_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR, 0));
  *fd_out = fd;
  return B200C_OK;
}
extern "C" int b200c_comm_mc_import(b200c_comm_t* c, int fd) {
  if (!c || fd < 0) return fail(B200C_EINVAL, "bad argument");
  if (!c->vmm) return fail(B200C_EUNSUPPORTED, "multicast needs the VMM share mode");
  DeviceGuard g(c->device);
  DRV(g_drv.MemImportFromShareableHandle(&c->mc_handle, (void*)(uintptr_t)fd, CU_MEM_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR));
  c->mc_have_handle = true;
  return B200C_OK;
}
extern "C" int b200c_comm_mc_add_device(b200c_comm_t* c) {
  if (!c || !c->mc_have_handle) return fail(B200C_ESTATE, "no multicast handle");
  DeviceGuard g(c->device);
  DRV(g_drv.MulticastAddDevice(c->mc_handle, c->cudev));
  c->mc_added = true;
  return B200C_OK;
}
extern "C" int b200c_comm_mc_bind(b200c_comm_t* c) {
  if (!c || !c->mc_added) return fail(B200C_ESTATE, "device not added to the multicast object");
  DeviceGuard g(c->device);
  DRV(g_drv.MulticastBindMem(c->mc_handle, 0, c->own_handle, 0, c->arena_bytes, 0));
  c->mc_bound = true;
  int rc = map_handle(c, c->mc_handle, &c->mc_arena);
  if (rc) { c->mc_arena = nullptr; return rc; }
  return B200C_OK;
}

extern "C" int b200c_comm_mc_disable(b200c_comm_t* c) {
  if (!c) return fail(B200C_EINVAL, "null communicator");
  DeviceGuard g(c->device);
  if (c->mc_arena) { g_drv.MemUnmap((CUdeviceptr)c->mc_arena, c->arena_bytes); g_drv.MemAddressFree((CUdeviceptr)c->mc_arena, c->arena_bytes); c->mc_arena = nullptr; }
  if (c->ready) c->dev.mc_arena = nullptr;
  return B200C_OK;
}

extern "C" int b200c_comm_ready(b200c_comm_t* c) {
  if (!c) return fail(B200C_EINVAL, "null communicator");
  if (c->destroyed) return fail(B200C_ESTATE, "communicator destroyed");
  for (int j = 0; j < c->world; j++)
    if (!c->imported[j]) return fail(B200C_ESTATE, "peer %d not imported yet", j);
  DevComm& d = c->dev;
  memset(&d, 0, sizeof d);
  d.rank = c->rank; d.world = c->world;
  for (int j = 0; j < c->world; j++) d.arena[j] = c->arena[j];
  d.mc_arena = c->mc_arena;
  d.status = c->status_dev;
  d.timeout_ns = (unsigned long long)c->cfg.timeout_ms * 1000000ull;
  d.staging_bytes = c->cfg.staging_bytes;
  d.off_staging = c->off_staging;
  d.off_p2p = c->off_p2p;
  d.p2p_cell_bytes = c->cfg.p2p_slot_bytes;
  d.p2p_cells = (int)c->cfg.p2p_slots;
  d.off_mring = c->off_mring;
  d.mcells = (int)c->mcells;
  d.off_ll = c->off_ll;
  d.ll_words = c->ll_words;
  // multicast: the root's payload leaves it once whatever the number of receivers, so it is chosen as soon as
  // there is more than one
  c->bcast_mc = c->world > 2;
  if (const char* e = getenv("B200COLL_BCAST_MULTICAST")) c->bcast_mc = e[0] == '1';
  c->ready = true;
  return B200C_OK;
}

extern "C" int b200c_comm_abort(b200c_comm_t* c) {
  if (!c) return fail(B200C_EINVAL, "null communicator");
  if (c->status_host) c->status_host->abort_flag = 1;
  return B200C_OK;
}

extern "C" int b200c_comm_check(b200c_comm_t* c) {
  if (!c) return fail(B200C_EINVAL, "null communicator");
  if (!c->status_host) return B200C_OK;
  int e = c->status_host->error;
  if (e == 0) return B200C_OK;
  static const char* const phases[] = {"arrive", "flagA", "flagB", "p2p-ready", "p2p-ack", "ll-slot"};  // by WaitPhase
  static_assert(sizeof(phases) / sizeof(phases[0]) == kNumWaitPhases, "one name per WaitPhase");
  int ph = c->status_host->err_phase;
  if (e == B200C_EMISMATCH)
    return fail(e, "%s: rank %d, op seq %u, peer %d announced signature %08x, this rank expected %08x", b200c_status_string(e), c->rank,
                c->status_host->err_seq, c->status_host->err_peer, c->status_host->err_a, c->status_host->err_b);
  return fail(e, "%s: rank %d, op seq %u, waiting on peer %d (%s)", b200c_status_string(e), c->rank, c->status_host->err_seq,
              c->status_host->err_peer, ph >= 0 && ph < kNumWaitPhases ? phases[ph] : "?");
}

extern "C" int b200c_comm_destroy(b200c_comm_t* c) {
  if (!c) return B200C_OK;
  if (c->destroyed) return B200C_OK;
  c->destroyed = true;
  c->ready = false;
  { std::lock_guard<std::mutex> lk(g_pool_mu); if (g_pool_comm == c) { g_pool_comm = nullptr; g_pool_nfree = 0; } }
  if (c->status_host) c->status_host->abort_flag = 1;
  DeviceGuard g(c->device);
  cudaDeviceSynchronize();
  cudaGetLastError();
  if (c->vmm) {
    if (c->mc_arena) { g_drv.MemUnmap((CUdeviceptr)c->mc_arena, c->arena_bytes); g_drv.MemAddressFree((CUdeviceptr)c->mc_arena, c->arena_bytes); }
    if (c->mc_bound && g_drv.MulticastUnbind) g_drv.MulticastUnbind(c->mc_handle, c->cudev, 0, c->arena_bytes);
    if (c->mc_have_handle) g_drv.MemRelease(c->mc_handle);
    for (int j = 0; j < c->world; j++) {
      if (!c->arena[j]) continue;
      g_drv.MemUnmap((CUdeviceptr)c->arena[j], c->arena_bytes);
      g_drv.MemAddressFree((CUdeviceptr)c->arena[j], c->arena_bytes);
      if (j != c->rank && c->peer_handle[j]) g_drv.MemRelease(c->peer_handle[j]);
    }
    if (c->own_handle) g_drv.MemRelease(c->own_handle);
  } else {
    for (int j = 0; j < c->world; j++) {
      if (!c->arena[j]) continue;
      if (j == c->rank) cudaFree(c->arena[j]);
      else cudaIpcCloseMemHandle(c->arena[j]);
    }
  }
  if (c->ps_in) { cudaStreamDestroy(c->ps_in); cudaStreamDestroy(c->ps_nv); cudaStreamDestroy(c->ps_out); cudaEventDestroy(c->pe_start);
    for (int i = 0; i < 8; i++) { if (c->pe_in[i]) cudaEventDestroy(c->pe_in[i]); if (c->pe_nv[i]) cudaEventDestroy(c->pe_nv[i]); if (c->pe_out[i]) cudaEventDestroy(c->pe_out[i]); } }
  if (c->status_host) cudaFreeHost((void*)c->status_host);
  c->status_host = nullptr;
  cudaGetLastError();
  delete c;
  return B200C_OK;
}

extern "C" int b200c_debug_fill_flags(b200c_comm_t* c, uint32_t value) {
  if (!c || c->destroyed) return fail(B200C_ESTATE, "communicator destroyed");
  DeviceGuard g(c->device);
  RT(cudaDeviceSynchronize());
  static_assert(kPadUsed % 4 == 0, "pad is u32 words");
  uint32_t* host = new uint32_t[kPadUsed / 4];
  for (size_t i = 0; i < kPadUsed / 4; i++) host[i] = value;
  cudaError_t e = cudaMemcpy(c->arena[c->rank], host, kPadUsed, cudaMemcpyHostToDevice);
  delete[] host;
  if (e != cudaSuccess) return fail(B200C_ECUDA, "cudaMemcpy failed: %s", cudaGetErrorString(e));
  // LL slots are matched by equality, not by >=: pre-stamp both halves with the flag of the NEXT LL op
  // (payload 0) so that exactly one LL launch can run without its peers
  size_t ll_u64 = 2 * (size_t)kMaxRanks * c->ll_words;
  if (ll_u64) {
    unsigned long long* h = new unsigned long long[ll_u64];
    for (size_t i = 0; i < ll_u64; i++) h[i] = (unsigned long long)(c->ll_seq + 1) << 32;
    e = cudaMemcpy(c->arena[c->rank] + c->off_ll, h, ll_u64 * 8, cudaMemcpyHostToDevice);
    delete[] h;
    if (e != cudaSuccess) return fail(B200C_ECUDA, "cudaMemcpy failed: %s", cudaGetErrorString(e));
  }
  return B200C_OK;
}

extern "C" int b200c_comm_rank(const b200c_comm_t* c) { return c ? c->rank : -1; }
extern "C" int b200c_comm_world(const b200c_comm_t* c) { return c ? c->world : -1; }
extern "C" int b200c_comm_has_multicast(const b200c_comm_t* c) { return c && c->mc_arena ? 1 : 0; }
extern "C" uint64_t b200c_comm_seq(const b200c_comm_t* c) { return c ? c->seq : 0; }
extern "C" void* b200c_comm_symmetric_base(b200c_comm_t* c) { return c && c->sym_bytes ? c->arena[c->rank] + c->off_sym : nullptr; }
extern "C" uint64_t b200c_comm_symmetric_bytes(const b200c_comm_t* c) { return c ? c->sym_bytes : 0; }

// ------------------------------------------------------------------------------------------------
// Symmetric pool: a torch.cuda.MemPool (CUDAPluggableAllocator) whose segments are carved out of one
// communicator's symmetric region, so ordinary torch tensors (and DDP's gradient buckets) allocated
// under `torch.cuda.use_mem_pool(pool)` are peer-mapped and multicast-bound: collectives on them take
// the zero-copy paths.  The allocator is deterministic (first fit over a sorted free list, 2 MiB
// granules): ranks that perform the same allocation sequence get the same offsets, which is what the
// symmetric paths require — and what b200c_allreduce verifies through the op signature (the offset is
// part of it), so a divergence is reported as EMISMATCH instead of reducing unrelated memory.
// ------------------------------------------------------------------------------------------------

extern "C" int b200c_pool_bind(b200c_comm_t* c) {
  std::lock_guard<std::mutex> lk(g_pool_mu);
  if (!c) { g_pool_comm = nullptr; g_pool_nfree = 0; return B200C_OK; }
  if (c->destroyed || !c->sym_bytes) return fail(B200C_ESTATE, "communicator has no symmetric region (config.symmetric_bytes)");
  g_pool_comm = c;
  g_pool_free[0] = PoolBlock{0, c->sym_bytes / kPoolGran * kPoolGran};
  g_pool_nfree = 1;
  return B200C_OK;
}
extern "C" void* b200c_pool_malloc(size_t size, int device, void* stream) {
  (void)stream;
  std::lock_guard<std::mutex> lk(g_pool_mu);
  b200c_comm* c = g_pool_comm;
  if (!c || c->destroyed || device != c->device || size == 0) return nullptr;
  size_t need = round_up(size, kPoolGran);
  for (int i = 0; i < g_pool_nfree; i++) {
    if (g_pool_free[i].len < need) continue;
    size_t off = g_pool_free[i].off;
    g_pool_free[i].off += need;
    g_pool_free[i].len -= need;
    if (g_pool_free[i].len == 0) { for (int j = i; j + 1 < g_pool_nfree; j++) g_pool_free[j] = g_pool_free[j + 1]; g_pool_nfree--; }
    return c->arena[c->rank] + c->off_sym + off;
  }
  return nullptr;  // torch reports the out-of-memory condition
}
extern "C" void b200c_pool_free(void* ptr, size_t size, int device, void* stream) {
  (void)device; (void)stream;
  std::lock_guard<std::mutex> lk(g_pool_mu);
  b200c_comm* c = g_pool_comm;
  if (!c || !ptr) return;
  char* base = c->arena[c->rank] + c->off_sym;
  if ((char*)ptr < base || (char*)ptr >= base + c->sym_bytes) return;
  size_t off = (size_t)((char*)ptr - base), len = round_up(size, kPoolGran);
  int i = 0;
  while (i < g_pool_nfree && g_pool_free[i].off < off) i++;
  if (g_pool_nfree >= 4095) return;  // cannot track it: leak the block rather than corrupt the list
  for (int j = g_pool_nfree; j > i; j--) g_pool_free[j] = g_pool_free[j - 1];
  g_pool_free[i] = PoolBlock{off, len};
  g_pool_nfree++;
  if (i + 1 < g_pool_nfree && g_pool_free[i].off + g_pool_free[i].len == g_pool_free[i + 1].off) {
    g_pool_free[i].len += g_pool_free[i + 1].len;
    for (int j = i + 1; j + 1 < g_pool_nfree; j++) g_pool_free[j] = g_pool_free[j + 1];
    g_pool_nfree--;
  }
  if (i > 0 && g_pool_free[i - 1].off + g_pool_free[i - 1].len == g_pool_free[i].off) {
    g_pool_free[i - 1].len += g_pool_free[i].len;
    for (int j = i; j + 1 < g_pool_nfree; j++) g_pool_free[j] = g_pool_free[j + 1];
    g_pool_nfree--;
  }
}

// ------------------------------------------------------------------------------------------------
// launch planning
// ------------------------------------------------------------------------------------------------
static int check_ready(b200c_comm* c) {
  if (!c) return fail(B200C_EINVAL, "null communicator");
  if (c->destroyed || !c->ready) return fail(B200C_ESTATE, "communicator not ready or destroyed");
  if (c->status_host->error) return b200c_comm_check(c);
  return B200C_OK;
}
// A launch that fails after its peers may already have launched the same op leaves this rank behind:
// poison the communicator so the failure is loud on every later call instead of a silent divergence.
static int launch_check(b200c_comm* c, const char* what) {
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) {
    if (c && c->status_host && c->status_host->error == 0) { c->status_host->error = B200C_ECUDA; c->status_host->err_seq = c->seq + 1; }
    return fail(B200C_ECUDA, "%s launch failed: %s", what, cudaGetErrorString(e));
  }
  g_launches.fetch_add(1);
  return B200C_OK;
}
// Block-cyclic plan for an extent of `units` elements (vector width `vec`).
//   small extents: one contiguous granule per block of at least min_tile_bytes (more blocks = lower latency);
//   large extents: fixed granule of `granule_bytes`, `max_blocks` blocks, each looping with stride grid * granule.
static void plan_tiles(size_t units, size_t elem_size, size_t vec, uint32_t max_blocks, size_t min_tile_bytes, size_t granule_bytes,
                       size_t* tile, int* grid) {
  if (units == 0) { *tile = vec; *grid = 1; return; }
  size_t bytes = units * elem_size;
  size_t nb = (bytes + min_tile_bytes - 1) / min_tile_bytes;
  if (nb < 1) nb = 1;
  if (nb > max_blocks) nb = max_blocks;
  size_t t = round_up((units + nb - 1) / nb, vec);
  if (t * elem_size > granule_bytes) t = granule_bytes / elem_size;  // granule_bytes is a multiple of 16 KiB, hence of vec
  size_t g = (units + t - 1) / t;
  *tile = t;
  *grid = (int)(g < max_blocks ? g : max_blocks);
}
// Plan for the round-pipelined kernels: at least ~4 rounds per block when the extent allows it, so that
// the software pipeline has something to overlap; granules of 8 KiB .. granule_bytes.
static void plan_rounds(size_t units, size_t elem_size, size_t vec, uint32_t max_blocks, size_t granule_bytes, size_t* tile, int* grid,
                        uint32_t* rounds) {
  size_t bytes = units * elem_size;
  size_t tb = bytes / ((size_t)max_blocks * 4) / 8192 * 8192;
  if (tb < 8192) tb = 8192;
  if (tb > granule_bytes) tb = granule_bytes;
  size_t t = tb / elem_size;
  (void)vec;
  size_t g = (units + t - 1) / t;
  if (g < 1) g = 1;
  *tile = t;
  *grid = (int)(g < max_blocks ? g : max_blocks);
  *rounds = (uint32_t)((units + (size_t)*grid * t - 1) / ((size_t)*grid * t));
}
static uint32_t make_sig(int opcode, int dtype, int op, size_t n, int root, int extra) {
  uint64_t h = 1469598103934665603ull;
  uint64_t v[6] = {(uint64_t)opcode, (uint64_t)dtype, (uint64_t)op, (uint64_t)n, (uint64_t)(root + 1), (uint64_t)extra};
  for (int i = 0; i < 6; i++) { h ^= v[i]; h *= 1099511628211ull; }
  return ((uint32_t)(h ^ (h >> 32)) & 0x7fffffffu) | 1u;  // never 0 and never the 0xFFFFFFFF wildcard
}
// The op takes sequence number seq + 1; the counters only advance once the launch has succeeded
// (commit_args), so a rejected call (EINVAL / EUNSUPPORTED before any launch) leaves the ranks aligned.
static void base_args(b200c_comm* c, CollArgs* a) {
  memset(a, 0, sizeof *a);
  a->c = c->dev;
  a->seq = c->seq + 1;
  a->root = -1;
}
// the only place where seq, pipe_base (by the op's round count) and ll_seq (LL ops carry the next one) advance
static void commit_args(b200c_comm* c, const CollArgs& a, uint32_t rounds = 0) {
  c->seq = a.seq;
  c->pipe_base += rounds;
  if (a.ll_seq) c->ll_seq = a.ll_seq;
}
// One collective over `total` units (elements, or bytes for the byte kernels), in pieces of at most `cap`.  For
// each piece, step(a, done, rounds) fills the CollArgs that base_args started (a.n comes in as the piece's extent
// and may be lowered), sets the round count of a round-pipelined kernel and launches.
template <typename Step>
static int run_pieces(b200c_comm* c, size_t total, size_t cap, const char* what, Step&& step) {
  for (size_t done = 0; done < total;) {
    CollArgs a;
    base_args(c, &a);
    a.n = total - done < cap ? total - done : cap;
    uint32_t rounds = 0;
    int rc = step(a, done, rounds);
    if (rc) return rc;
    rc = launch_check(c, what);
    if (rc) return rc;
    commit_args(c, a, rounds);
    done += a.n;
  }
  return B200C_OK;
}
// one rank: the result is the input, copied unless the call is in place
static int copy_if_distinct(const void* src, void* dst, size_t bytes, cudaStream_t s) {
  if (src != dst) RT(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToDevice, s));
  return B200C_OK;
}
static int launch_same_type(int dtype, int kind, int op, const CollArgs& a, int grid, cudaStream_t s) {
  switch (dtype) {
    case B200C_INT8: return launch_i8(kind, op, a, grid, s);
    case B200C_UINT8: return launch_u8(kind, op, a, grid, s);
    case B200C_INT32: return launch_i32(kind, op, a, grid, s);
    case B200C_UINT32: return launch_u32(kind, op, a, grid, s);
    case B200C_INT64: return launch_i64(kind, op, a, grid, s);
    case B200C_UINT64: return launch_u64(kind, op, a, grid, s);
    case B200C_FLOAT16: return launch_f16(kind, op, a, grid, s);
    case B200C_FLOAT32: return launch_f32(kind, op, a, grid, s);
    case B200C_FLOAT64: return launch_f64(kind, op, a, grid, s);
    case B200C_BFLOAT16: return launch_bf16(kind, op, a, grid, s);
    default: return fail(B200C_EUNSUPPORTED, "dtype %d", dtype);
  }
}

enum { OPC_ALLREDUCE = 1, OPC_REDUCE, OPC_BROADCAST, OPC_ALLGATHER, OPC_REDUCESCATTER, OPC_BARRIER };
constexpr size_t kMinTileBytes = 8192;

// The fused-mean family's (buffer dtype, wire dtype) pairs: f32 on an f32, bf16 or f16 wire, and bf16 / f16
// on their own.  Calls f(Type<TI>{}, Type<TW>{}) for the pair and returns false for any other.
template <typename T>
struct Type { using type = T; };
template <typename F>
static bool with_scaled_types(int dtype, int wire, F&& f) {
  switch (dtype * 16 + wire) {
    case B200C_FLOAT32 * 16 + B200C_FLOAT32: f(Type<float>{}, Type<float>{}); return true;
    case B200C_FLOAT32 * 16 + B200C_BFLOAT16: f(Type<float>{}, Type<bf16_t>{}); return true;
    case B200C_FLOAT32 * 16 + B200C_FLOAT16: f(Type<float>{}, Type<f16_t>{}); return true;
    case B200C_BFLOAT16 * 16 + B200C_BFLOAT16: f(Type<bf16_t>{}, Type<bf16_t>{}); return true;
    case B200C_FLOAT16 * 16 + B200C_FLOAT16: f(Type<f16_t>{}, Type<f16_t>{}); return true;
    default: return false;
  }
}
constexpr int kScaledPairs[][2] = {{B200C_FLOAT32, B200C_FLOAT32}, {B200C_FLOAT32, B200C_BFLOAT16}, {B200C_FLOAT32, B200C_FLOAT16},
                                   {B200C_BFLOAT16, B200C_BFLOAT16}, {B200C_FLOAT16, B200C_FLOAT16}};

// mixed-type (bucket dtype != wire dtype) and NVLS launches live in this TU
template <typename TI, typename TW>
static void launch_mixed(int algo, const CollArgs& a, int grid, cudaStream_t s) {
  with_world_t(a.c.world, [&](auto wt) {
    constexpr int WT = decltype(wt)::value;
    if (algo == B200C_ALGO_ONESHOT) k_allreduce_oneshot<TI, TW, B200C_SUM, WT><<<grid, kThreads, 0, s>>>(a);
    else k_allreduce_twoshot<TI, TW, B200C_SUM, WT><<<grid, kThreads, 0, s>>>(a);
  });
}
static void launch_rs_scaled(int dtype, int wire, const CollArgs& a, int grid, cudaStream_t s) {
  with_scaled_types(dtype, wire, [&](auto ti, auto tw) {
    with_world_t(a.c.world, [&](auto wt) {
      k_reducescatter_scaled<typename decltype(ti)::type, typename decltype(tw)::type, decltype(wt)::value><<<grid, kThreads, 0, s>>>(a);
    });
  });
}
static void launch_nvls(int dtype, int wire, const CollArgs& a, int grid, cudaStream_t s, bool pipe, bool lanes = false) {
  with_scaled_types(dtype, wire, [&](auto ti, auto tw) {
    using TI = typename decltype(ti)::type;
    using TW = typename decltype(tw)::type;
    if (lanes) k_allreduce_nvls_lanes<TI, TW><<<grid, kThreads, 0, s>>>(a);
    else if (pipe) k_allreduce_nvls_rounds<TI, TW><<<grid, kThreads, 0, s>>>(a);
    else k_allreduce_nvls<TI, TW><<<grid, kThreads, 0, s>>>(a);
  });
}
template <typename TI, typename TW>
static int local_scale_grid(b200c_comm* c, size_t bytes) {
  // no peers to wait for, so the grid is sized for HBM: one CTA per 32 KiB, but never more CTAs than are
  // resident at once (a second, partial wave would idle part of the chip for a whole pass)
  if (c->local_scale_ctas_per_sm == 0) {
    int nb = 0;
    if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&nb, k_local_scale<float, bf16_t>, kThreads, 0) != cudaSuccess || nb < 1) { cudaGetLastError(); nb = 2; }
    c->local_scale_ctas_per_sm = nb;
  }
  size_t want = (bytes + 32767) / 32768, cap = (size_t)c->sm_count * c->local_scale_ctas_per_sm;
  return (int)(want < 1 ? 1 : (want > cap ? cap : want));
}

// ------------------------------------------------------------------------------------------------
// Multi-stream staged NVLS (the largest plain tensors).  Instead of one kernel that interleaves local copies
// with switch traffic, the message is cut into pieces and every piece runs three ordinary kernels on three
// internal streams, chained by events:
//     copy-in(i)  [user -> staging region i % R, any grid]      on ps_in
//     switch(i)   [the 32-CTA zero-copy NVLS kernel on region]  on ps_nv   (the only kernel that waits for peers)
//     copy-out(i) [region -> user]                              on ps_out
// so copy-in(i+1) and copy-out(i-1) overlap switch(i), the switch kernel keeps its few CTAs streaming, and the
// copies are plain full-speed local kernels that never spin.  A barrier op opens the pipeline (every peer has
// finished what it did before, so both staging halves are free to serve as R regions) and another one closes it
// on the caller's stream after the last copy-out (no later op of a peer can touch this rank's staging while a
// copy-out still reads it).  Region reuse: copy-in(i+R) waits for copy-out(i); every peer finished reducing
// region i before switch(i) completed (flag B).
// ------------------------------------------------------------------------------------------------
// Copy n elements from the caller's buffer (dtype) into a staging region (wire), or back (OUT, which bypasses
// L2).  A 2-byte payload on its own wire is a plain copy: the bf16 kernel serves f16 as well.
template <bool OUT>
static void launch_stage_copy(int dtype, int wire, const void* src, void* dst, size_t n, int sm_count, cudaStream_t s) {
  with_scaled_types(dtype, wire, [&](auto ti, auto tw) {
    constexpr bool plain = sizeof(typename decltype(ti)::type) == 2;
    using TI = std::conditional_t<plain, bf16_t, typename decltype(ti)::type>;
    using TW = std::conditional_t<plain, bf16_t, typename decltype(tw)::type>;
    using TS = std::conditional_t<OUT, TW, TI>;
    using TD = std::conditional_t<OUT, TI, TW>;
    size_t tile = kStageTileBytes / (sizeof(TS) > sizeof(TD) ? sizeof(TS) : sizeof(TD));
    size_t want = (n + tile - 1) / tile, cap = (size_t)sm_count * 4;
    int grid = (int)(want < 1 ? 1 : (want > cap ? cap : want));
    k_stage_copy<TS, TD, OUT><<<grid, kThreads, 0, s>>>(static_cast<const TS*>(src), static_cast<TD*>(dst), n);
  });
}
static int pipeline_setup(b200c_comm* c) {
  if (c->ps_in) return B200C_OK;
  int lo = 0, hi = 0;
  RT(cudaDeviceGetStreamPriorityRange(&lo, &hi));
  RT(cudaStreamCreateWithPriority(&c->ps_in, cudaStreamNonBlocking, lo));
  RT(cudaStreamCreateWithPriority(&c->ps_nv, cudaStreamNonBlocking, hi));   // the switch kernel's CTAs go first
  RT(cudaStreamCreateWithPriority(&c->ps_out, cudaStreamNonBlocking, lo));
  RT(cudaEventCreateWithFlags(&c->pe_start, cudaEventDisableTiming));
  for (int i = 0; i < 8; i++) {
    RT(cudaEventCreateWithFlags(&c->pe_in[i], cudaEventDisableTiming));
    RT(cudaEventCreateWithFlags(&c->pe_nv[i], cudaEventDisableTiming));
    RT(cudaEventCreateWithFlags(&c->pe_out[i], cudaEventDisableTiming));
  }
  return B200C_OK;
}
// Lazy module loading (CUDA_MODULE_LOADING=LAZY, torch's default) loads a kernel at its first launch, and the load
// can wait for the kernels already running in the context.  A kernel that waits for a peer's kernel in the same
// context -- a receive posted before the matching send on another stream, the ranks of a loopback world -- then
// waits for a launch that waits for it, until timeout_ms.  So the first communicator of a device loads every kernel
// that waits for a peer before any of them runs, and the batch-norm kernels that a sync batch norm launches between
// its collectives.  (tests/test_gpu_zz_schedules.py posts receives first.)
static int load_kernels(int device) {
  static std::mutex mu;
  static uint32_t loaded = 0;   // bit d: device d is done
  std::lock_guard<std::mutex> lk(mu);
  if (device < 32 && ((loaded >> device) & 1)) return B200C_OK;
  int rc = B200C_OK;
  auto load = [&](auto kernel) { if (!rc) rc = load_kernel(kernel); };
  CollArgs a;
  memset(&a, 0, sizeof a);
  for (int world : {2, 3, 4, 8}) {   // 3 stands for every world size taken at run time (WT = 0)
    a.c.world = world;
    for (int dt = 0; dt < B200C_NUM_DTYPES; dt++)
      for (int op : {B200C_SUM, B200C_PROD, B200C_MAX, B200C_MIN})
        if (!rc) rc = launch_same_type(dt, KIND_LOAD, op, a, 0, nullptr);
    with_world_t(world, [&](auto wt) {
      constexpr int WT = decltype(wt)::value;
      load(k_allreduce_oneshot<float, bf16_t, B200C_SUM, WT>);
      load(k_allreduce_twoshot<float, bf16_t, B200C_SUM, WT>);
      load(k_allreduce_oneshot<float, f16_t, B200C_SUM, WT>);
      load(k_allreduce_twoshot<float, f16_t, B200C_SUM, WT>);
      for (const auto& p : kScaledPairs)
        with_scaled_types(p[0], p[1], [&](auto ti, auto tw) {
          load(k_reducescatter_scaled<typename decltype(ti)::type, typename decltype(tw)::type, WT>);
        });
    });
  }
  for (const auto& p : kScaledPairs)
    with_scaled_types(p[0], p[1], [&](auto ti, auto tw) {
      using TI = typename decltype(ti)::type;
      using TW = typename decltype(tw)::type;
      load(k_allreduce_nvls<TI, TW>);
      load(k_allreduce_nvls_rounds<TI, TW>);
      load(k_allreduce_nvls_lanes<TI, TW>);
    });
  load(k_allgather);
  load(k_broadcast);
  load(k_broadcast_rounds);
  load(k_barrier);
  load(k_send);
  load(k_send_multi);
  load(k_recv);
  // the sync batch norm's kernels run between collectives on the ranks' streams
  if (!rc && bn::load_kernels() != cudaSuccess) rc = B200C_ECUDA;
  if (rc) return fail(rc, "loading the collective kernels failed: %s", cudaGetErrorString(cudaGetLastError()));
  if (device < 32) loaded |= 1u << device;
  return B200C_OK;
}
static int barrier_op(b200c_comm* c, cudaStream_t s) {
  CollArgs a;
  base_args(c, &a);
  a.sig = make_sig(OPC_BARRIER, 0, 0, 0, -1, 0);
  k_barrier<<<1, 32, 0, s>>>(a);
  int rc = launch_check(c, "barrier");
  if (rc) return rc;
  commit_args(c, a);
  return B200C_OK;
}
static int allreduce_streams(b200c_comm* c, const void* send, void* recv, size_t count, int dtype, int wire, int op, float scale,
                             int has_scale, cudaStream_t user) {
  (void)op;
  const int W = c->world;
  const size_t esz = b200c_dtype_size(dtype), wsz = b200c_dtype_size(wire), vec = 16 / wsz;
  int rc = pipeline_setup(c);
  if (rc) return rc;
  size_t piece_bytes = c->cfg.nvls_streams_piece_bytes;
  size_t area = 2 * c->cfg.staging_bytes;
  while (area / piece_bytes < 3 && piece_bytes > (1u << 20)) piece_bytes /= 2;
  int R = (int)(area / piece_bytes);
  if (R < 3) return fail(B200C_EINVAL, "staging_bytes too small for the multi-stream pipeline");
  if (R > 8) R = 8;
  const size_t piece_elems = piece_bytes / wsz / (vec * W) * (vec * W);
  // Piece sizes: the pipeline's fill (first copy-in) and drain (last copy-out) are not overlapped with anything, so
  // the first and the last piece are a quarter of the regular size.
  const size_t small = piece_elems / 4 / (vec * W) * (vec * W);
  const uint32_t cap = c->cfg.nvls_blocks && c->cfg.nvls_blocks < c->cfg.max_blocks ? c->cfg.nvls_blocks : c->cfg.max_blocks;
  // open: every peer has finished its previous op, so the whole staging area is ours to partition
  rc = barrier_op(c, user);
  if (rc) return rc;
  RT(cudaEventRecord(c->pe_start, user));
  RT(cudaStreamWaitEvent(c->ps_in, c->pe_start, 0));
  size_t e0 = 0;
  int last_reg = 0;
  for (int i = 0; e0 < count; i++) {
    const int reg = i % R;
    last_reg = reg;
    const size_t left = count - e0;
    size_t n;
    if (small && count > 2 * piece_elems) {
      if (i == 0) n = small;
      else if (left <= small) n = left;
      else if (left <= piece_elems + small) n = left - small;   // the piece before the short last one takes the remainder
      else n = piece_elems;
    } else {
      n = left < piece_elems ? left : piece_elems;
    }
    char* region = c->arena[c->rank] + c->off_staging + (size_t)reg * piece_bytes;
    const char* src = static_cast<const char*>(send) + e0 * esz;
    char* dst = static_cast<char*>(recv) + e0 * esz;
    if (i >= R) RT(cudaStreamWaitEvent(c->ps_in, c->pe_out[reg], 0));   // the region's previous piece has been copied out
    launch_stage_copy<false>(dtype, wire, src, region, n, c->sm_count, c->ps_in);
    rc = launch_check(c, "stage_in");
    if (rc) return rc;
    RT(cudaEventRecord(c->pe_in[reg], c->ps_in));
    RT(cudaStreamWaitEvent(c->ps_nv, c->pe_in[reg], 0));
    CollArgs a;
    base_args(c, &a);
    a.in = region; a.out = region;
    a.has_scale = has_scale; a.scale = scale;
    a.n = n;
    a.chunk = round_up((n + W - 1) / W, vec);
    a.symmetric = 1;
    a.sym_off = (size_t)(region - c->arena[c->rank]);
    int grid;
    plan_tiles(a.chunk, wsz, vec, cap, kMinTileBytes, c->cfg.granule_bytes, &a.tile, &grid);
    a.sig = make_sig(OPC_ALLREDUCE, dtype * 16 + wire, B200C_SUM, n, reg, B200C_ALGO_NVLS_STREAMS * 8 + i % 8);
    launch_nvls(wire, wire, a, grid, c->ps_nv, false);
    rc = launch_check(c, "nvls(stream pipeline)");
    if (rc) return rc;
    commit_args(c, a);
    RT(cudaEventRecord(c->pe_nv[reg], c->ps_nv));
    RT(cudaStreamWaitEvent(c->ps_out, c->pe_nv[reg], 0));
    launch_stage_copy<true>(dtype, wire, region, dst, n, c->sm_count, c->ps_out);
    rc = launch_check(c, "stage_out");
    if (rc) return rc;
    RT(cudaEventRecord(c->pe_out[reg], c->ps_out));
    e0 += n;
  }
  // close: the caller's stream continues after the last copy-out, and peers only move on after this rank got here
  RT(cudaStreamWaitEvent(user, c->pe_out[last_reg], 0));
  return barrier_op(c, user);
}

// One rank: no peers, so only the wire rounding and the scale remain.
static int allreduce_local(b200c_comm* c, const void* send, void* recv, size_t count, int dtype, int wire, float scale, int has_scale,
                           cudaStream_t s) {
  const size_t esz = b200c_dtype_size(dtype);
  if (!has_scale && wire == dtype) return copy_if_distinct(send, recv, count * esz, s);
  CollArgs a; memset(&a, 0, sizeof a);
  a.c = c->dev; a.in = send; a.out = recv; a.n = count; a.has_scale = has_scale; a.scale = scale;
  // Large, 16-byte aligned buffers stream through shared memory with the bulk copy engine (TMA); the
  // plain LSU kernel takes small buffers, unaligned views and the sub-tile tail.
  if (count * esz >= (1u << 20) && ((uintptr_t)send & 15) == 0 && ((uintptr_t)recv & 15) == 0 &&
      (dtype == B200C_FLOAT32 || ((dtype == B200C_BFLOAT16 || dtype == B200C_FLOAT16) && wire == dtype))) {
    size_t ntiles = count * esz / kTmaTileBytes;
    size_t tma_elems = ntiles * kTmaTileBytes / esz;
    if (c->tma_ctas_per_sm == 0) {
      int nb = 0;
      for (const auto& p : kScaledPairs)
        with_scaled_types(p[0], p[1], [](auto ti, auto tw) {
          cudaFuncSetAttribute(k_local_scale_tma<typename decltype(ti)::type, typename decltype(tw)::type>,
                               cudaFuncAttributeMaxDynamicSharedMemorySize, kTmaSmemBytes);
        });
      if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&nb, k_local_scale_tma<float, bf16_t>, kTmaThreads, kTmaSmemBytes) != cudaSuccess || nb < 1) { cudaGetLastError(); nb = 1; }
      c->tma_ctas_per_sm = nb;
    }
    // as many CTAs as are resident at once (measured: a smaller "balanced" grid of 384 x 5 tiles is slower, 13.7 vs
    // 12.9 us per 30 MiB bucket — what counts is how many bulk loads are in flight from the first microsecond)
    size_t cap = (size_t)c->sm_count * c->tma_ctas_per_sm;
    int tgrid = (int)(ntiles < cap ? ntiles : cap);
    with_scaled_types(dtype, wire, [&](auto ti, auto tw) {
      k_local_scale_tma<typename decltype(ti)::type, typename decltype(tw)::type><<<tgrid, kTmaThreads, kTmaSmemBytes, s>>>(a);
    });
    int rc = launch_check(c, "local_scale_tma");
    if (rc) return rc;
    if (tma_elems == count) return B200C_OK;
    a.in = static_cast<const char*>(send) + tma_elems * esz;
    a.out = static_cast<char*>(recv) + tma_elems * esz;
    a.n = count - tma_elems;
  }
  int grid = local_scale_grid<float, bf16_t>(c, a.n * esz);
  if (dtype == B200C_FLOAT64) k_local_scale<double, double><<<grid, kThreads, 0, s>>>(a);
  else if (!with_scaled_types(dtype, wire, [&](auto ti, auto tw) {
             k_local_scale<typename decltype(ti)::type, typename decltype(tw)::type><<<grid, kThreads, 0, s>>>(a);
           }))
    return copy_if_distinct(send, recv, count * esz, s);  // integer AVG over one rank is the identity
  return launch_check(c, "local_scale");
}

// AUTO picks per piece, from the bytes left; the NVLS variants are NVLS pieces planned as pipelined or lanes.
static int choose_algo(b200c_comm* c, int algo, size_t total_bytes, size_t bytes_left, bool ll_ok, bool nvls_ok, bool in_sym,
                       bool* pipe, bool* lanes) {
  const int W = c->world;
  int al = algo;
  if (al == B200C_ALGO_NVLS_PIPE) { al = B200C_ALGO_NVLS; *pipe = true; }
  if (al == B200C_ALGO_NVLS_LANES) { al = B200C_ALGO_NVLS; *lanes = true; }
  if (al == B200C_ALGO_AUTO) {
    if (ll_ok && total_bytes <= c->cfg.ll_max_bytes) al = B200C_ALGO_LL;
    else if (bytes_left <= c->cfg.oneshot_max_bytes) al = B200C_ALGO_ONESHOT;
    else if (nvls_ok && W > 2 && bytes_left >= c->cfg.nvls_min_bytes && (W >= 6 || in_sym)) al = B200C_ALGO_NVLS;  // W = 4: two-shot beats staged NVLS
    else al = B200C_ALGO_TWOSHOT;
  }
  return al;
}

// The planners below set the piece's extent (a.n, at most `left` elements), chunk, tile and grid.
static void plan_ll(b200c_comm* c, CollArgs& a, size_t left, size_t esz, size_t vec, int& grid) {
  size_t n = left;
  a.chunk = round_up(n, vec);
  a.tile = vec;
  a.ll_seq = c->ll_seq + 1;
  size_t nvec = (n * esz + 15) / 16;
  size_t nb = (nvec + kLLThreads - 1) / kLLThreads;
  grid = (int)(nb < 1 ? 1 : (nb > c->cfg.max_blocks ? c->cfg.max_blocks : nb));
  a.n = n;
}
static void plan_oneshot(b200c_comm* c, CollArgs& a, size_t left, size_t wsz, size_t vec, int& grid) {
  const int W = c->world;
  size_t cap = c->cfg.staging_bytes / W / wsz / vec * vec;  // elements per slot
  size_t n = left < cap ? left : cap;
  a.chunk = round_up(n, vec);
  plan_tiles(n, wsz, vec, c->cfg.max_blocks, kMinTileBytes, c->cfg.granule_bytes, &a.tile, &grid);
  a.n = n;
}
static void plan_twoshot(b200c_comm* c, CollArgs& a, size_t left, size_t wsz, size_t vec, int& grid) {
  const int W = c->world;
  size_t cap_chunk = c->cfg.staging_bytes / W / wsz / vec * vec;
  size_t cap = cap_chunk * W;
  size_t n = left < cap ? left : cap;
  a.chunk = round_up((n + W - 1) / W, vec);
  plan_tiles(a.chunk, wsz, vec, c->cfg.max_blocks, kMinTileBytes, c->cfg.granule_bytes, &a.tile, &grid);
  a.n = n;
}
// NVLS: zero-copy on a symmetric buffer (`sym`), else staged: plain, round-pipelined (`pipe`) or lanes (`lanes`),
// the latter two also chosen here for AUTO by size.
static int plan_nvls(b200c_comm* c, CollArgs& a, size_t left, size_t wsz, size_t vec, bool sym, int algo, bool& pipe, bool& lanes,
                     int& grid, uint32_t& rounds) {
  const int W = c->world;
  // the zero-copy kernel is pure switch traffic (few CTAs are best); the staged kernels also do the local copies
  const uint32_t nvls_sym_cap = c->cfg.nvls_blocks && c->cfg.nvls_blocks < c->cfg.max_blocks ? c->cfg.nvls_blocks : c->cfg.max_blocks;
  // symmetric buffers need no staging; pieces of at most 256 MiB keep the peers' TLB reach
  size_t cap = sym ? ((size_t)256 << 20) / wsz : c->cfg.staging_bytes / wsz / vec * vec;
  size_t n = left < cap ? left : cap;
  a.chunk = round_up((n + W - 1) / W, vec);
  a.symmetric = sym ? 1 : 0;
  a.sym_off = sym ? (size_t)((const char*)a.in - c->arena[c->rank]) : 0;
  if (!sym && algo == B200C_ALGO_AUTO && c->cfg.nvls_lanes_min_bytes && left * wsz >= c->cfg.nvls_lanes_min_bytes) lanes = true;
  if (!sym && !lanes && algo == B200C_ALGO_AUTO && c->cfg.nvls_pipe_min_bytes && n * wsz >= c->cfg.nvls_pipe_min_bytes) pipe = true;
  if (sym) pipe = lanes = false;  // nothing to overlap: the symmetric path has no staging copies
  if (lanes) {
    // the ring is rewritten every three rounds, so the staging capacity does not bound the piece: take it all
    n = left;
    a.chunk = round_up((n + W - 1) / W, vec);
    uint32_t L = c->cfg.nvls_lanes;
    uint32_t Kc = c->cfg.max_blocks / L - 1;
    if (Kc > 7) Kc = 7;
    if (Kc < 1) Kc = 1;
    // granule: the configured size, smaller for messages that would otherwise give a lane fewer than ~4 rounds
    size_t tb = c->cfg.lane_granule_bytes, chunk_bytes = a.chunk * wsz;
    size_t want = chunk_bytes / ((size_t)L * 4) / 8192 * 8192;
    if (want < 8192) want = 8192;
    if (tb > want) tb = want;
    size_t ring = (size_t)L * kLaneSlots * W * tb;
    while (ring > c->cfg.staging_bytes && tb > 8192) { tb -= 8192; ring = (size_t)L * kLaneSlots * W * tb; }
    while (ring > c->cfg.staging_bytes && L > 1) { L--; ring = (size_t)L * kLaneSlots * W * tb; }   // a small staging area: fewer lanes
    if (ring > c->cfg.staging_bytes) return fail(B200C_EINVAL, "staging_bytes too small for the lane kernel's ring (%zu bytes)", ring);
    a.tile = tb / wsz;
    a.lane_copy = (int)Kc;
    size_t ngran = (a.chunk + a.tile - 1) / a.tile;
    uint32_t used = (uint32_t)(ngran < L ? ngran : L);   // lanes that own at least one granule
    grid = (int)(used * (1 + Kc));
    rounds = (uint32_t)((ngran + used - 1) / used);
    a.pipe_base = c->pipe_base;
  } else if (pipe) {
    plan_rounds(a.chunk, wsz, vec, c->cfg.max_blocks, c->cfg.granule_bytes, &a.tile, &grid, &rounds);
    a.pipe_base = c->pipe_base;
  } else {
    plan_tiles(a.chunk, wsz, vec, sym ? nvls_sym_cap : c->cfg.max_blocks, kMinTileBytes, c->cfg.granule_bytes, &a.tile, &grid);
  }
  a.n = n;
  return B200C_OK;
}

static int allreduce_impl(b200c_comm* c, const void* send, void* recv, size_t count, int dtype, int wire, int op, float scale,
                          int has_scale, int algo, cudaStream_t s) {
  int rc = check_ready(c);
  if (rc) return rc;
  size_t esz = b200c_dtype_size(dtype), wsz = b200c_dtype_size(wire);
  if (!esz || !wsz) return fail(B200C_EINVAL, "bad dtype %d / wire %d", dtype, wire);
  if (op < 0 || op >= B200C_NUM_OPS) return fail(B200C_EINVAL, "bad reduce op %d", op);
  if (count && (!send || !recv)) return fail(B200C_EINVAL, "null buffer");
  if (wire != dtype) {
    if (!(dtype == B200C_FLOAT32 && (wire == B200C_BFLOAT16 || wire == B200C_FLOAT16))) return fail(B200C_EUNSUPPORTED, "wire dtype %d for buffer dtype %d", wire, dtype);
    if (op != B200C_SUM && op != B200C_AVG) return fail(B200C_EUNSUPPORTED, "compressed wire supports SUM/AVG only");
  }
  if (algo < B200C_ALGO_AUTO || algo > B200C_ALGO_NVLS_STREAMS) return fail(B200C_EINVAL, "bad algo %d", algo);
  if (op == B200C_AVG) { has_scale = 1; scale = 1.f / (float)c->world; }
  if (count == 0) return B200C_OK;
  DeviceGuard g(c->device);
  const int W = c->world;
  const size_t vec = 16 / wsz;
  if (W == 1) return allreduce_local(c, send, recv, count, dtype, wire, scale, has_scale, s);

  const bool nvls_ok = c->mc_arena && (op == B200C_SUM || op == B200C_AVG) &&
                       (wire == B200C_FLOAT32 || wire == B200C_BFLOAT16 || wire == B200C_FLOAT16);
  if ((algo == B200C_ALGO_NVLS || algo == B200C_ALGO_NVLS_PIPE || algo == B200C_ALGO_NVLS_LANES || algo == B200C_ALGO_NVLS_STREAMS) && !nvls_ok) return fail(B200C_EUNSUPPORTED, "NVLS needs a bound multicast object, SUM/AVG and f32/bf16/f16");
  const bool ll_ok = wire == dtype && c->ll_words && count * esz <= c->ll_words * 4;
  if (algo == B200C_ALGO_LL && !ll_ok) return fail(B200C_EUNSUPPORTED, "LL needs wire == dtype and at most %zu bytes (ll_max_bytes)", c->ll_words * 4);
  const char* in = static_cast<const char*>(send);
  char* out = static_cast<char*>(recv);
  // in place, same dtype on the wire, inside the symmetric region: eligible for the zero-copy path
  bool in_sym = false;
  if (wire == dtype && send == recv && c->sym_bytes && (((uintptr_t)send) & 15) == 0 && (count * esz) % 16 == 0) {
    const char* base = c->arena[c->rank] + c->off_sym;
    in_sym = in >= base && in + count * esz <= base + c->sym_bytes;
  }
  if (!in_sym && (algo == B200C_ALGO_NVLS_STREAMS ||
                  (algo == B200C_ALGO_AUTO && nvls_ok && W >= 6 && c->cfg.nvls_streams_min_bytes && count * wsz >= c->cfg.nvls_streams_min_bytes)))
    return allreduce_streams(c, send, recv, count, dtype, wire, op, scale, has_scale, s);
  // each algorithm's planner sizes its own pieces
  return run_pieces(c, count, count, "allreduce", [&](CollArgs& a, size_t done, uint32_t& rounds) -> int {
    const size_t left = count - done;
    bool pipe = false, lanes = false;
    const int al = choose_algo(c, algo, count * esz, left * wsz, ll_ok, nvls_ok, in_sym, &pipe, &lanes);
    a.in = in + done * esz; a.out = out + done * esz;
    a.has_scale = has_scale; a.scale = scale;
    // symmetric zero-copy NVLS: buffer lives in the symmetric region at the same offset everywhere
    const bool sym = al == B200C_ALGO_NVLS && in_sym;
    int grid = 0;  // set by every planner that returns B200C_OK
    if (al == B200C_ALGO_LL) plan_ll(c, a, left, esz, vec, grid);
    else if (al == B200C_ALGO_ONESHOT) plan_oneshot(c, a, left, wsz, vec, grid);
    else if (al == B200C_ALGO_TWOSHOT) plan_twoshot(c, a, left, wsz, vec, grid);
    else {
      int rc = plan_nvls(c, a, left, wsz, vec, sym, algo, pipe, lanes, grid, rounds);
      if (rc) return rc;
    }
    // a symmetric buffer must sit at the same arena offset on every rank: the offset is part of the signature
    a.sig = make_sig(OPC_ALLREDUCE, dtype * 16 + wire, op, a.n, sym ? (int)((a.sym_off >> 4) & 0x3fffffff) : -1, al * 8 + (sym ? 1 : 0) + (pipe ? 2 : 0) + (lanes ? 4 : 0));
    if (al == B200C_ALGO_NVLS) launch_nvls(dtype, wire, a, grid, s, pipe, lanes);
    else if (wire != dtype) {
      if (wire == B200C_BFLOAT16) launch_mixed<float, bf16_t>(al, a, grid, s);
      else launch_mixed<float, f16_t>(al, a, grid, s);
    } else {
      int kind = al == B200C_ALGO_LL ? KIND_LL : (al == B200C_ALGO_ONESHOT ? KIND_ONESHOT : KIND_TWOSHOT);
      return launch_same_type(dtype, kind, op, a, grid, s);
    }
    return B200C_OK;
  });
}

extern "C" int b200c_allreduce(b200c_comm_t* c, const void* send, void* recv, size_t count, int dtype, int op, int algo,
                               b200c_stream_t stream) {
  // AVG on integers: SUM then truncating divide by world (ncclAvg semantics); handled by apply_scale.
  return allreduce_impl(c, send, recv, count, dtype, dtype, op, 1.f, 0, algo, (cudaStream_t)stream);
}

extern "C" int b200c_allreduce_scaled(b200c_comm_t* c, const void* send, void* recv, size_t count, int dtype, int wire_dtype,
                                      float scale, int algo, b200c_stream_t stream) {
  if (dtype != B200C_FLOAT32 && dtype != B200C_BFLOAT16 && dtype != B200C_FLOAT16)
    return fail(B200C_EUNSUPPORTED, "scaled allreduce supports f32/bf16/f16 buffers, got %d", dtype);
  return allreduce_impl(c, send, recv, count, dtype, wire_dtype, B200C_SUM, scale, 1, algo, (cudaStream_t)stream);
}

extern "C" int b200c_reduce(b200c_comm_t* c, const void* send, void* recv, size_t count, int dtype, int op, int root,
                            b200c_stream_t stream) {
  int rc = check_ready(c);
  if (rc) return rc;
  size_t esz = b200c_dtype_size(dtype);
  if (!esz) return fail(B200C_EINVAL, "bad dtype %d", dtype);
  if (op < 0 || op >= B200C_NUM_OPS) return fail(B200C_EINVAL, "bad reduce op %d", op);
  if (root < 0 || root >= c->world) return fail(B200C_EINVAL, "bad root %d", root);
  if (count == 0) return B200C_OK;
  if (!send || (c->rank == root && !recv)) return fail(B200C_EINVAL, "null buffer");
  cudaStream_t s = (cudaStream_t)stream;
  DeviceGuard g(c->device);
  if (c->world == 1) return copy_if_distinct(send, recv, count * esz, s);
  const size_t vec = 16 / esz;
  size_t cap = c->cfg.staging_bytes / c->world / esz / vec * vec;
  return run_pieces(c, count, cap, "reduce", [&](CollArgs& a, size_t done, uint32_t&) {
    a.in = static_cast<const char*>(send) + done * esz;
    a.out = recv ? static_cast<char*>(recv) + done * esz : nullptr;
    a.chunk = round_up(a.n, vec); a.root = root;
    if (op == B200C_AVG) { a.has_scale = 1; a.scale = 1.f / c->world; }
    int grid;
    plan_tiles(a.n, esz, vec, c->cfg.max_blocks, kMinTileBytes, c->cfg.granule_bytes, &a.tile, &grid);
    a.sig = make_sig(OPC_REDUCE, dtype, op, a.n, root, 0);
    return launch_same_type(dtype, KIND_REDUCE, op, a, grid, s);
  });
}

extern "C" int b200c_reducescatter(b200c_comm_t* c, const void* const* send_ptrs, void* recv, size_t count, int dtype, int op,
                                   b200c_stream_t stream) {
  int rc = check_ready(c);
  if (rc) return rc;
  size_t esz = b200c_dtype_size(dtype);
  if (!esz) return fail(B200C_EINVAL, "bad dtype %d", dtype);
  if (op < 0 || op >= B200C_NUM_OPS) return fail(B200C_EINVAL, "bad reduce op %d", op);
  if (count == 0) return B200C_OK;
  if (!send_ptrs || !recv) return fail(B200C_EINVAL, "null buffer");
  for (int j = 0; j < c->world; j++) if (!send_ptrs[j]) return fail(B200C_EINVAL, "send_ptrs[%d] is null", j);
  cudaStream_t s = (cudaStream_t)stream;
  DeviceGuard g(c->device);
  if (c->world == 1) return copy_if_distinct(send_ptrs[0], recv, count * esz, s);
  const size_t vec = 16 / esz;
  size_t cap = c->cfg.staging_bytes / c->world / esz / vec * vec;
  return run_pieces(c, count, cap, "reducescatter", [&](CollArgs& a, size_t done, uint32_t&) {
    for (int j = 0; j < c->world; j++) a.in_ptrs[j] = static_cast<const char*>(send_ptrs[j]) + done * esz;
    a.out = static_cast<char*>(recv) + done * esz;
    a.chunk = round_up(a.n, vec);
    if (op == B200C_AVG) { a.has_scale = 1; a.scale = 1.f / c->world; }
    int grid;
    plan_tiles(a.n, esz, vec, c->cfg.max_blocks, kMinTileBytes, c->cfg.granule_bytes, &a.tile, &grid);
    a.sig = make_sig(OPC_REDUCESCATTER, dtype, op, a.n, -1, 0);
    return launch_same_type(dtype, KIND_REDUCESCATTER, op, a, grid, s);
  });
}

extern "C" int b200c_reducescatter_scaled(b200c_comm_t* c, const void* const* send_ptrs, void* recv, size_t count, int dtype,
                                          int wire_dtype, float scale, b200c_stream_t stream) {
  int rc = check_ready(c);
  if (rc) return rc;
  if (dtype != B200C_FLOAT32 && dtype != B200C_BFLOAT16 && dtype != B200C_FLOAT16)
    return fail(B200C_EUNSUPPORTED, "scaled reducescatter supports f32/bf16/f16 buffers, got %d", dtype);
  const size_t esz = b200c_dtype_size(dtype), wsz = b200c_dtype_size(wire_dtype);
  if (!wsz) return fail(B200C_EINVAL, "bad wire dtype %d", wire_dtype);
  if (wire_dtype != dtype && !(dtype == B200C_FLOAT32 && (wire_dtype == B200C_BFLOAT16 || wire_dtype == B200C_FLOAT16)))
    return fail(B200C_EUNSUPPORTED, "wire dtype %d for buffer dtype %d", wire_dtype, dtype);
  if (count == 0) return B200C_OK;
  if (!send_ptrs || !recv) return fail(B200C_EINVAL, "null buffer");
  for (int j = 0; j < c->world; j++) if (!send_ptrs[j]) return fail(B200C_EINVAL, "send_ptrs[%d] is null", j);
  cudaStream_t s = (cudaStream_t)stream;
  // one rank: only the wire rounding and the scale remain, which is the one-rank scaled allreduce
  if (c->world == 1) return allreduce_impl(c, send_ptrs[0], recv, count, dtype, wire_dtype, B200C_SUM, scale, 1, B200C_ALGO_AUTO, s);
  DeviceGuard g(c->device);
  const size_t vec = 16 / wsz;
  size_t cap = c->cfg.staging_bytes / c->world / wsz / vec * vec;   // pieces are sized in wire bytes
  return run_pieces(c, count, cap, "reducescatter_scaled", [&](CollArgs& a, size_t done, uint32_t&) {
    for (int j = 0; j < c->world; j++) a.in_ptrs[j] = static_cast<const char*>(send_ptrs[j]) + done * esz;
    a.out = static_cast<char*>(recv) + done * esz;
    a.chunk = round_up(a.n, vec);
    a.has_scale = 1; a.scale = scale;
    int grid;
    plan_tiles(a.n, wsz, vec, c->cfg.max_blocks, kMinTileBytes, c->cfg.granule_bytes, &a.tile, &grid);
    // the wire is part of the signature: a peer in a plain reducescatter (or on another wire) is a mismatch
    a.sig = make_sig(OPC_REDUCESCATTER, dtype, B200C_SUM, a.n, -1, 16 + wire_dtype);
    launch_rs_scaled(dtype, wire_dtype, a, grid, s);
    return B200C_OK;
  });
}

extern "C" int b200c_allgather(b200c_comm_t* c, const void* send, void* const* recv_ptrs, size_t count, int dtype,
                               b200c_stream_t stream) {
  int rc = check_ready(c);
  if (rc) return rc;
  size_t esz = b200c_dtype_size(dtype);
  if (!esz) return fail(B200C_EINVAL, "bad dtype %d", dtype);
  if (count == 0) return B200C_OK;
  if (!send || !recv_ptrs) return fail(B200C_EINVAL, "null buffer");
  for (int j = 0; j < c->world; j++) if (!recv_ptrs[j]) return fail(B200C_EINVAL, "recv_ptrs[%d] is null", j);
  cudaStream_t s = (cudaStream_t)stream;
  DeviceGuard g(c->device);
  size_t bytes = count * esz;
  if (c->world == 1) return copy_if_distinct(send, recv_ptrs[0], bytes, s);
  size_t cap = c->cfg.staging_bytes / c->world / 16 * 16;
  return run_pieces(c, bytes, cap, "allgather", [&](CollArgs& a, size_t done, uint32_t&) {
    a.in = static_cast<const char*>(send) + done;
    for (int j = 0; j < c->world; j++) a.out_ptrs[j] = static_cast<char*>(recv_ptrs[j]) + done;
    a.chunk = round_up(a.n, 16);
    int grid;
    plan_tiles(a.n, 1, 16, c->cfg.max_blocks, kMinTileBytes, c->cfg.granule_bytes, &a.tile, &grid);
    a.sig = make_sig(OPC_ALLGATHER, dtype, 0, a.n, -1, 0);
    k_allgather<<<grid, kThreads, 0, s>>>(a);
    return B200C_OK;
  });
}

// ------------------------------------------------------------------------------------------------
// fused batch norm (norm_kernels.cuh, launched by inst_norm.cu): a local site runs two kernels per direction; a sync
// site runs the local phases around b200c_allgather and b200c_allreduce
// ------------------------------------------------------------------------------------------------
extern "C" size_t b200c_bn_scratch_bytes(int channels) {
  return channels < 1 || channels > bn::kMaxChannels ? 0 : bn::scratch_bytes(channels);
}

extern "C" size_t b200c_bn_sync_scratch_bytes(int channels, int world) {
  return channels < 1 || channels > bn::kMaxChannels || world < 1 || world > kMaxRanks ? 0 : bn::sync_scratch_bytes(channels, world);
}

static const char* bn_site(bool sync) { return sync ? "sync batch norm" : "batch norm"; }

// Checks shared by every call.  min_m is 1 for a local site and 0 for a sync site, where a rank may have no rows.  A
// site without ReLU has no identity (forward) or gradient for it (backward), no mask and no second gradient.  The
// mask holds 8 channels per byte of a row, so it takes C % 8 == 0 only.
static int check_bn(const char* site, int min_m, int m, int c, const void* scratch, int relu, const void* mask, const void* residual,
                    const void* dy2) {
  if (m < min_m || c < 1 || c > bn::kMaxChannels || (int64_t)m * c > INT32_MAX)
    return fail(B200C_EINVAL, "%s: bad shape m=%d c=%d", site, m, c);
  if (!scratch) return fail(B200C_EINVAL, "%s: null scratch", site);
  if (!relu && (mask || residual || dy2)) return fail(B200C_EINVAL, "%s: a site without ReLU takes no mask, identity or dy2", site);
  if (mask && c % 8) return fail(B200C_EINVAL, "%s mask: channels=%d is not a multiple of 8", site, c);
  return B200C_OK;
}

// All arguments are checked before the communicator and before any launch.  A sync rank without rows launches only
// the merge.
static int bn_forward(b200c_comm_t* comm, bool sync, const void* x, const void* identity, void* y, void* mask, int relu,
                      const float* weight, const float* bias, float* running_mean, float* running_var, int64_t* num_batches_tracked,
                      float* save_mean, float* save_invstd, float* norm_fct, int m, int channels, float momentum, float eps,
                      void* scratch, b200c_stream_t stream) {
  int rc = check_bn(bn_site(sync), sync ? 0 : 1, m, channels, scratch, relu, mask, identity, nullptr);
  if (rc) return rc;
  if ((m && (!x || !y)) || !weight || !bias || !running_mean || !running_var || !save_mean || !save_invstd || (sync && !norm_fct))
    return fail(B200C_EINVAL, "%s forward: null buffer", bn_site(sync));
  const bn::FwdArgs a{x, identity, y, mask, relu != 0, weight, bias, running_mean, running_var,
                      reinterpret_cast<long long*>(num_batches_tracked), save_mean, save_invstd, m, channels, momentum, eps, scratch};
  cudaStream_t s = (cudaStream_t)stream;
  if (!sync) {
    RT(bn::forward(a, s));
    g_launches.fetch_add(2);
    return B200C_OK;
  }
  rc = check_ready(comm);
  if (rc) return rc;
  DeviceGuard g(comm->device);
  const int rows = m != 0;
  RT(bn::sync_stats(a, s));
  g_launches.fetch_add(rows);
  const bn::SyncRows r = bn::sync_rows(scratch, channels);
  void* gathered[kMaxRanks];
  for (int j = 0; j < comm->world; j++) gathered[j] = r.gathered + j * r.row_floats;
  rc = b200c_allgather(comm, r.local, gathered, (size_t)2 * channels + 1, B200C_FLOAT32, stream);
  if (rc) return rc;
  RT(bn::sync_apply(a, comm->world, norm_fct, s));
  g_launches.fetch_add(1 + rows);
  return B200C_OK;
}

static int bn_backward(b200c_comm_t* comm, bool sync, const void* dy, const void* dy2, const void* y, const void* mask, int relu,
                       const void* x, void* dy_masked, void* dx, const float* weight, const float* save_mean, const float* save_invstd,
                       const float* norm_fct, float* grad_weight, float* grad_bias, int m, int channels, void* scratch,
                       b200c_stream_t stream) {
  int rc = check_bn(bn_site(sync), sync ? 0 : 1, m, channels, scratch, relu, mask, dy_masked, dy2);
  if (rc) return rc;
  if ((m && (!dy || !x || !dx || (relu && !y && !mask))) || !weight || !save_mean || !save_invstd || (sync && !norm_fct) ||
      !grad_weight || !grad_bias)
    return fail(B200C_EINVAL, "%s backward: null buffer", bn_site(sync));
  const bn::BwdArgs a{dy, dy2, y, mask, x, dy_masked, dx, relu != 0, weight, save_mean, save_invstd, norm_fct, grad_weight, grad_bias,
                      m, channels, scratch};
  cudaStream_t s = (cudaStream_t)stream;
  if (!sync) {
    RT(bn::backward(a, s));
    g_launches.fetch_add(2);
    return B200C_OK;
  }
  rc = check_ready(comm);
  if (rc) return rc;
  DeviceGuard g(comm->device);
  const int rows = m != 0;
  RT(bn::sync_bwd_reduce(a, s));
  g_launches.fetch_add(rows);
  float* sums = bn::sync_rows(scratch, channels).sums;
  rc = b200c_allreduce(comm, sums, sums, (size_t)2 * channels, B200C_FLOAT32, B200C_SUM, B200C_ALGO_AUTO, stream);
  if (rc) return rc;
  RT(bn::sync_bwd_elemt(a, s));
  g_launches.fetch_add(rows);
  return B200C_OK;
}

extern "C" int b200c_bn_forward(const void* x, const void* identity, void* y, const float* weight, const float* bias,
                                float* running_mean, float* running_var, int64_t* num_batches_tracked, float* save_mean,
                                float* save_invstd, int m, int channels, float momentum, float eps, void* scratch,
                                b200c_stream_t stream) {
  return bn_forward(nullptr, false, x, identity, y, nullptr, 1, weight, bias, running_mean, running_var, num_batches_tracked, save_mean,
                    save_invstd, nullptr, m, channels, momentum, eps, scratch, stream);
}

extern "C" int b200c_bn_forward_mask(const void* x, const void* identity, void* y, uint8_t* mask, const float* weight,
                                     const float* bias, float* running_mean, float* running_var, int64_t* num_batches_tracked,
                                     float* save_mean, float* save_invstd, int m, int channels, float momentum, float eps,
                                     void* scratch, b200c_stream_t stream) {
  if (!mask) return fail(B200C_EINVAL, "batch norm mask: null mask");
  return bn_forward(nullptr, false, x, identity, y, mask, 1, weight, bias, running_mean, running_var, num_batches_tracked, save_mean,
                    save_invstd, nullptr, m, channels, momentum, eps, scratch, stream);
}

extern "C" int b200c_bn_sync_forward(b200c_comm_t* comm, const void* x, const void* identity, void* y, uint8_t* mask, int relu,
                                     const float* weight, const float* bias, float* running_mean, float* running_var,
                                     int64_t* num_batches_tracked, float* save_mean, float* save_invstd, float* norm_fct, int m,
                                     int channels, float momentum, float eps, void* scratch, b200c_stream_t stream) {
  return bn_forward(comm, true, x, identity, y, mask, relu, weight, bias, running_mean, running_var, num_batches_tracked, save_mean,
                    save_invstd, norm_fct, m, channels, momentum, eps, scratch, stream);
}

extern "C" int b200c_bn_backward(const void* dy, const void* y, const void* x, void* dy_masked, void* dx, const float* weight,
                                 const float* save_mean, const float* save_invstd, float* grad_weight, float* grad_bias, int m,
                                 int channels, void* scratch, b200c_stream_t stream) {
  return bn_backward(nullptr, false, dy, nullptr, y, nullptr, 1, x, dy_masked, dx, weight, save_mean, save_invstd, nullptr, grad_weight,
                     grad_bias, m, channels, scratch, stream);
}

extern "C" int b200c_bn_backward_mask(const void* dy, const void* dy2, const uint8_t* mask, const void* x, void* dy_masked,
                                      void* dx, const float* weight, const float* save_mean, const float* save_invstd,
                                      float* grad_weight, float* grad_bias, int m, int channels, void* scratch,
                                      b200c_stream_t stream) {
  if (!mask) return fail(B200C_EINVAL, "batch norm mask: null mask");
  return bn_backward(nullptr, false, dy, dy2, nullptr, mask, 1, x, dy_masked, dx, weight, save_mean, save_invstd, nullptr, grad_weight,
                     grad_bias, m, channels, scratch, stream);
}

extern "C" int b200c_bn_sync_backward(b200c_comm_t* comm, const void* dy, const void* dy2, const void* y, const uint8_t* mask, int relu,
                                      const void* x, void* dy_masked, void* dx, const float* weight, const float* save_mean,
                                      const float* save_invstd, const float* norm_fct, float* grad_weight, float* grad_bias, int m,
                                      int channels, void* scratch, b200c_stream_t stream) {
  return bn_backward(comm, true, dy, dy2, y, mask, relu, x, dy_masked, dx, weight, save_mean, save_invstd, norm_fct, grad_weight,
                     grad_bias, m, channels, scratch, stream);
}

// A tail whose identity is a downsample branch's batch norm.
extern "C" size_t b200c_bn_dual_scratch_bytes(int channels) {
  return channels < 1 || channels > bn::kMaxChannels / 2 ? 0 : bn::dual_scratch_bytes(channels);
}

static int check_dual(int channels) {
  if (channels > bn::kMaxChannels / 2) return fail(B200C_EINVAL, "batch norm dual: channels=%d above %d", channels, bn::kMaxChannels / 2);
  return B200C_OK;
}

extern "C" int b200c_bn_forward_dual(const void* x, const void* x_ds, void* y, uint8_t* mask, const float* weight, const float* bias,
                                     float* running_mean, float* running_var, int64_t* num_batches_tracked, float* save_mean,
                                     float* save_invstd, float momentum, float eps, const float* weight_ds, const float* bias_ds,
                                     float* running_mean_ds, float* running_var_ds, int64_t* num_batches_tracked_ds,
                                     float* save_mean_ds, float* save_invstd_ds, float momentum_ds, float eps_ds, int m, int channels,
                                     void* scratch, b200c_stream_t stream) {
  int rc = check_bn("batch norm dual", 1, m, channels, scratch, 1, mask, x_ds, nullptr);
  if (!rc) rc = check_dual(channels);
  if (rc) return rc;
  if (!x || !x_ds || !y || !weight || !bias || !running_mean || !running_var || !save_mean || !save_invstd || !weight_ds ||
      !bias_ds || !running_mean_ds || !running_var_ds || !save_mean_ds || !save_invstd_ds)
    return fail(B200C_EINVAL, "batch norm dual forward: null buffer");
  const bn::FwdArgs a{x, nullptr, y, mask, true, weight, bias, running_mean, running_var,
                      reinterpret_cast<long long*>(num_batches_tracked), save_mean, save_invstd, m, channels, momentum, eps, scratch};
  const bn::FwdArgs b{x_ds, nullptr, nullptr, nullptr, false, weight_ds, bias_ds, running_mean_ds, running_var_ds,
                      reinterpret_cast<long long*>(num_batches_tracked_ds), save_mean_ds, save_invstd_ds, m, channels, momentum_ds,
                      eps_ds, scratch};
  RT(bn::forward_dual(a, b, (cudaStream_t)stream));
  g_launches.fetch_add(2);
  return B200C_OK;
}

extern "C" int b200c_bn_backward_dual(const void* dy, const void* dy2, const void* y, const uint8_t* mask, const void* x,
                                      const void* x_ds, void* dx, void* dx_ds, const float* weight, const float* save_mean,
                                      const float* save_invstd, float* grad_weight, float* grad_bias, const float* weight_ds,
                                      const float* save_mean_ds, const float* save_invstd_ds, float* grad_weight_ds,
                                      float* grad_bias_ds, int m, int channels, void* scratch, b200c_stream_t stream) {
  int rc = check_bn("batch norm dual", 1, m, channels, scratch, 1, mask, nullptr, dy2);
  if (!rc) rc = check_dual(channels);
  if (rc) return rc;
  if (!dy || (!y && !mask) || !x || !x_ds || !dx || !dx_ds || !weight || !save_mean || !save_invstd || !grad_weight || !grad_bias ||
      !weight_ds || !save_mean_ds || !save_invstd_ds || !grad_weight_ds || !grad_bias_ds)
    return fail(B200C_EINVAL, "batch norm dual backward: null buffer");
  const bn::BwdArgs a{dy, dy2, mask ? nullptr : y, mask, x, nullptr, dx, true, weight, save_mean, save_invstd, nullptr, grad_weight,
                      grad_bias, m, channels, scratch};
  const bn::BwdArgs b{nullptr, nullptr, nullptr, nullptr, x_ds, nullptr, dx_ds, false, weight_ds, save_mean_ds, save_invstd_ds, nullptr,
                      grad_weight_ds, grad_bias_ds, m, channels, scratch};
  RT(bn::backward_dual(a, b, (cudaStream_t)stream));
  g_launches.fetch_add(2);
  return B200C_OK;
}

// The stem: n images of h x w rows.  The shape is checked in 64 bits before it becomes the site's m.
static int check_pool(const char* dir, int n, int h, int w, int channels, int* m) {
  if (n < 1 || h < 1 || w < 1 || (int64_t)n * h * w > INT32_MAX)
    return fail(B200C_EINVAL, "batch norm pool %s: bad shape n=%d h=%d w=%d c=%d", dir, n, h, w, channels);
  *m = n * h * w;
  return B200C_OK;
}

extern "C" int b200c_bn_forward_pool(const void* x, void* y, uint8_t* argmax, const float* weight, const float* bias,
                                     float* running_mean, float* running_var, int64_t* num_batches_tracked, float* save_mean,
                                     float* save_invstd, int n, int h, int w, int channels, float momentum, float eps, void* scratch,
                                     b200c_stream_t stream) {
  int m = 0;
  int rc = check_pool("forward", n, h, w, channels, &m);
  if (!rc) rc = check_bn("batch norm pool", 1, m, channels, scratch, 1, nullptr, nullptr, nullptr);
  if (rc) return rc;
  if (!x || !y || !argmax || !weight || !bias || !running_mean || !running_var || !save_mean || !save_invstd)
    return fail(B200C_EINVAL, "batch norm pool forward: null buffer");
  bn::FwdArgs a{x, nullptr, y, nullptr, true, weight, bias, running_mean, running_var,
                reinterpret_cast<long long*>(num_batches_tracked), save_mean, save_invstd, m, channels, momentum, eps, scratch};
  a.argmax = argmax;
  a.pool_h = h;
  a.pool_w = w;
  RT(bn::forward(a, (cudaStream_t)stream));
  g_launches.fetch_add(2);
  return B200C_OK;
}

extern "C" int b200c_bn_backward_pool(const void* dy, const uint8_t* argmax, const void* x, void* g, void* dx, const float* weight,
                                      const float* save_mean, const float* save_invstd, float* grad_weight, float* grad_bias, int n,
                                      int h, int w, int channels, void* scratch, b200c_stream_t stream) {
  int m = 0;
  int rc = check_pool("backward", n, h, w, channels, &m);
  if (!rc) rc = check_bn("batch norm pool", 1, m, channels, scratch, 1, nullptr, nullptr, nullptr);
  if (rc) return rc;
  if (!dy || !argmax || !x || !g || !dx || !weight || !save_mean || !save_invstd || !grad_weight || !grad_bias)
    return fail(B200C_EINVAL, "batch norm pool backward: null buffer");
  bn::BwdArgs a{dy, nullptr, nullptr, nullptr, x, g, dx, true, weight, save_mean, save_invstd, nullptr, grad_weight, grad_bias,
                m, channels, scratch};
  a.argmax = argmax;
  a.pool_h = h;
  a.pool_w = w;
  RT(bn::backward(a, (cudaStream_t)stream));
  g_launches.fetch_add(2);
  return B200C_OK;
}

// Eval mode (norm_infer.cuh): one kernel per site.  An eval batch norm takes one value per channel (m >= 1).
static int check_infer(const char* site, int param_bf16, int m, int c) {
  if (m < 1 || c < 1 || (int64_t)m * c > INT32_MAX) return fail(B200C_EINVAL, "%s: bad shape m=%d c=%d", site, m, c);
  if (param_bf16 != 0 && param_bf16 != 1) return fail(B200C_EINVAL, "%s: param_bf16=%d is neither 0 nor 1", site, param_bf16);
  return B200C_OK;
}

static int run_infer(const bn::InferArgs& a, b200c_stream_t stream) {
  RT(bn::infer(a, (cudaStream_t)stream));
  g_launches.fetch_add(1);
  return B200C_OK;
}

extern "C" int b200c_bn_infer(const void* x, const void* identity, void* y, const void* weight, const void* bias,
                              const void* running_mean, const void* running_var, int param_bf16, float eps, int m, int channels,
                              b200c_stream_t stream) {
  int rc = check_infer("batch norm infer", param_bf16, m, channels);
  if (rc) return rc;
  if (!x || !y || !weight || !bias || !running_mean || !running_var) return fail(B200C_EINVAL, "batch norm infer: null buffer");
  return run_infer({x, identity, y, {weight, bias, running_mean, running_var, eps}, {}, false, param_bf16 != 0, m, channels, 0, 0},
                   stream);
}

extern "C" int b200c_bn_infer_dual(const void* x, const void* x_ds, void* y, const void* weight, const void* bias,
                                   const void* running_mean, const void* running_var, float eps, const void* weight_ds,
                                   const void* bias_ds, const void* running_mean_ds, const void* running_var_ds, float eps_ds,
                                   int param_bf16, int m, int channels, b200c_stream_t stream) {
  int rc = check_infer("batch norm infer dual", param_bf16, m, channels);
  if (rc) return rc;
  if (!x || !x_ds || !y || !weight || !bias || !running_mean || !running_var || !weight_ds || !bias_ds || !running_mean_ds ||
      !running_var_ds)
    return fail(B200C_EINVAL, "batch norm infer dual: null buffer");
  return run_infer({x, x_ds, y, {weight, bias, running_mean, running_var, eps}, {weight_ds, bias_ds, running_mean_ds, running_var_ds, eps_ds},
                    true, param_bf16 != 0, m, channels, 0, 0},
                   stream);
}

extern "C" int b200c_bn_infer_pool(const void* x, void* y, const void* weight, const void* bias, const void* running_mean,
                                   const void* running_var, int param_bf16, float eps, int n, int h, int w, int channels,
                                   b200c_stream_t stream) {
  int m = 0;
  int rc = check_pool("infer", n, h, w, channels, &m);
  if (!rc) rc = check_infer("batch norm infer pool", param_bf16, m, channels);
  if (rc) return rc;
  if (!x || !y || !weight || !bias || !running_mean || !running_var) return fail(B200C_EINVAL, "batch norm infer pool: null buffer");
  return run_infer({x, nullptr, y, {weight, bias, running_mean, running_var, eps}, {}, false, param_bf16 != 0, m, channels, h, w}, stream);
}

// VGG's stage end, max_pool2d(relu(bn(x)), 2, 2) (norm_pool2.cuh): n images of h x w rows, h and w at least 2 (torch's
// max_pool2d refuses an output of zero rows or columns), channels 1..kMaxChannels, n * h * w * channels below 2^31, and
// every bf16 operand on its 2-byte grid and every fp32 one on its 4-byte grid (the kernels run 8 channels per thread
// where all of them are also on the 16-byte grid and channels % 8 == 0, else 1).
static int check_pool2(const char* site, int n, int h, int w, int c, int* m) {
  if (n < 1 || h < 2 || w < 2 || c < 1 || c > bn::kMaxChannels || (int64_t)n * h * w * c > INT32_MAX)
    return fail(B200C_EINVAL, "%s: bad shape n=%d h=%d w=%d channels=%d", site, n, h, w, c);
  *m = n * h * w;
  return B200C_OK;
}

static int check_grid(const char* site, std::initializer_list<const void*> bf16s, std::initializer_list<const void*> fp32s) {
  for (const void* q : bf16s)
    if (reinterpret_cast<uintptr_t>(q) % 2) return fail(B200C_EINVAL, "%s: a bf16 operand is off the 2-byte grid", site);
  for (const void* q : fp32s)
    if (reinterpret_cast<uintptr_t>(q) % 4) return fail(B200C_EINVAL, "%s: an fp32 operand is off the 4-byte grid", site);
  return B200C_OK;
}

extern "C" int b200c_bn_forward_pool2(const void* x, void* y, uint8_t* argmax, const float* weight, const float* bias,
                                      float* running_mean, float* running_var, int64_t* num_batches_tracked, float* save_mean,
                                      float* save_invstd, int n, int h, int w, int channels, float momentum, float eps, void* scratch,
                                      b200c_stream_t stream) {
  const char* site = "batch norm pool2 forward";
  if (!x || !y || !argmax || !weight || !bias || !running_mean || !running_var || !save_mean || !save_invstd || !scratch)
    return fail(B200C_EINVAL, "%s: null buffer", site);
  int m = 0;
  int rc = check_pool2(site, n, h, w, channels, &m);
  if (!rc) rc = check_grid(site, {x, y}, {weight, bias, running_mean, running_var, save_mean, save_invstd});
  if (!rc && reinterpret_cast<uintptr_t>(num_batches_tracked) % 8)
    rc = fail(B200C_EINVAL, "%s: num_batches_tracked is off the 8-byte grid", site);
  if (rc) return rc;
  bn::FwdArgs a{x, nullptr, y, nullptr, true, weight, bias, running_mean, running_var,
                reinterpret_cast<long long*>(num_batches_tracked), save_mean, save_invstd, m, channels, momentum, eps, scratch};
  a.argmax = argmax;
  a.pool_h = h;
  a.pool_w = w;
  RT(bn::forward_pool2(a, (cudaStream_t)stream));
  g_launches.fetch_add(2);
  return B200C_OK;
}

extern "C" int b200c_bn_backward_pool2(const void* dy, const uint8_t* argmax, const void* x, void* dx, const float* weight,
                                       const float* save_mean, const float* save_invstd, float* grad_weight, float* grad_bias, int n,
                                       int h, int w, int channels, void* scratch, b200c_stream_t stream) {
  const char* site = "batch norm pool2 backward";
  if (!dy || !argmax || !x || !dx || !weight || !save_mean || !save_invstd || !grad_weight || !grad_bias || !scratch)
    return fail(B200C_EINVAL, "%s: null buffer", site);
  int m = 0;
  int rc = check_pool2(site, n, h, w, channels, &m);
  if (!rc) rc = check_grid(site, {dy, x, dx}, {weight, save_mean, save_invstd, grad_weight, grad_bias});
  if (rc) return rc;
  bn::BwdArgs a{dy, nullptr, nullptr, nullptr, x, nullptr, dx, true, weight, save_mean, save_invstd, nullptr, grad_weight, grad_bias,
                m, channels, scratch};
  a.argmax = argmax;
  a.pool_h = h;
  a.pool_w = w;
  RT(bn::backward_pool2(a, (cudaStream_t)stream));
  g_launches.fetch_add(2);
  return B200C_OK;
}

extern "C" int b200c_bn_infer_pool2(const void* x, void* y, const void* weight, const void* bias, const void* running_mean,
                                    const void* running_var, int param_bf16, float eps, int n, int h, int w, int channels,
                                    b200c_stream_t stream) {
  const char* site = "batch norm infer pool2";
  if (!x || !y || !weight || !bias || !running_mean || !running_var) return fail(B200C_EINVAL, "%s: null buffer", site);
  int m = 0;
  int rc = check_pool2(site, n, h, w, channels, &m);
  if (!rc) rc = check_infer(site, param_bf16, m, channels);
  if (!rc) rc = param_bf16 ? check_grid(site, {x, y, weight, bias, running_mean, running_var}, {})
                           : check_grid(site, {x, y}, {weight, bias, running_mean, running_var});
  if (rc) return rc;
  RT(bn::infer_pool2({x, nullptr, y, {weight, bias, running_mean, running_var, eps}, {}, false, param_bf16 != 0, m, channels, h, w},
                     (cudaStream_t)stream));
  g_launches.fetch_add(1);
  return B200C_OK;
}

// A batch norm followed by ReLU6, SiLU or Hardswish (norm_act.cuh): the local site's checks, an activation the kernels
// have, and (the eval site too) at most kMaxChannels channels.
static int check_act(const char* site, int act, int c) {
  if (!bn::act_ok(act)) return fail(B200C_EINVAL, "%s: unknown act=%d", site, act);
  if (c > bn::kMaxChannels) return fail(B200C_EINVAL, "%s: channels=%d above %d", site, c, bn::kMaxChannels);
  return B200C_OK;
}

extern "C" int b200c_bn_forward_act(const void* x, void* y, const float* weight, const float* bias, float* running_mean,
                                    float* running_var, int64_t* num_batches_tracked, float* save_mean, float* save_invstd, int act,
                                    int m, int channels, float momentum, float eps, void* scratch, b200c_stream_t stream) {
  int rc = check_bn("batch norm act", 1, m, channels, scratch, 1, nullptr, nullptr, nullptr);
  if (!rc) rc = check_act("batch norm act", act, channels);
  if (rc) return rc;
  if (!x || !y || !weight || !bias || !running_mean || !running_var || !save_mean || !save_invstd)
    return fail(B200C_EINVAL, "batch norm act forward: null buffer");
  const bn::FwdArgs a{x, nullptr, y, nullptr, false, weight, bias, running_mean, running_var,
                      reinterpret_cast<long long*>(num_batches_tracked), save_mean, save_invstd, m, channels, momentum, eps, scratch};
  RT(bn::forward_act(a, act, (cudaStream_t)stream));
  g_launches.fetch_add(2);
  return B200C_OK;
}

extern "C" int b200c_bn_backward_act(const void* dy, const void* x, void* g, void* dx, const float* weight, const float* bias,
                                     const float* save_mean, const float* save_invstd, float* grad_weight, float* grad_bias, int act,
                                     int m, int channels, void* scratch, b200c_stream_t stream) {
  int rc = check_bn("batch norm act", 1, m, channels, scratch, 1, nullptr, nullptr, nullptr);
  if (!rc) rc = check_act("batch norm act", act, channels);
  if (rc) return rc;
  if (!dy || !x || !g || !dx || !weight || !bias || !save_mean || !save_invstd || !grad_weight || !grad_bias)
    return fail(B200C_EINVAL, "batch norm act backward: null buffer");
  const bn::BwdArgs a{dy, nullptr, nullptr, nullptr, x, g, dx, false, weight, save_mean, save_invstd, nullptr, grad_weight, grad_bias,
                      m, channels, scratch};
  RT(bn::backward_act(a, bias, act, (cudaStream_t)stream));
  g_launches.fetch_add(2);
  return B200C_OK;
}

extern "C" int b200c_bn_infer_act(const void* x, void* y, const void* weight, const void* bias, const void* running_mean,
                                  const void* running_var, int param_bf16, float eps, int act, int m, int channels,
                                  b200c_stream_t stream) {
  int rc = check_infer("batch norm infer act", param_bf16, m, channels);
  if (!rc) rc = check_act("batch norm infer act", act, channels);
  if (rc) return rc;
  if (!x || !y || !weight || !bias || !running_mean || !running_var) return fail(B200C_EINVAL, "batch norm infer act: null buffer");
  RT(bn::infer_act({x, nullptr, y, {weight, bias, running_mean, running_var, eps}, {}, false, param_bf16 != 0, m, channels, 0, 0}, act,
                   (cudaStream_t)stream));
  g_launches.fetch_add(1);
  return B200C_OK;
}

// A batch norm followed by a residual add, with or without stochastic depth (norm_res.cuh): the local site's checks,
// at most kMaxChannels channels, noise only with an identity (forward) and rows_per_sample >= 1 dividing m with noise.
static int check_res(const char* site, int m, int c, const void* identity, const void* noise, int rows_per_sample) {
  if (c > bn::kMaxChannels) return fail(B200C_EINVAL, "%s: channels=%d above %d", site, c, bn::kMaxChannels);
  if (noise && !identity) return fail(B200C_EINVAL, "%s: noise without an identity", site);
  if (noise && (rows_per_sample < 1 || m % rows_per_sample))
    return fail(B200C_EINVAL, "%s: rows_per_sample=%d does not divide m=%d", site, rows_per_sample, m);
  return B200C_OK;
}

extern "C" int b200c_bn_forward_res(const void* x, const void* identity, const void* noise, int rows_per_sample, void* y,
                                    const float* weight, const float* bias, float* running_mean, float* running_var,
                                    int64_t* num_batches_tracked, float* save_mean, float* save_invstd, int m, int channels,
                                    float momentum, float eps, void* scratch, b200c_stream_t stream) {
  int rc = check_bn("batch norm res", 1, m, channels, scratch, 1, nullptr, nullptr, nullptr);
  if (!rc) rc = check_res("batch norm res", m, channels, identity, noise, rows_per_sample);
  if (rc) return rc;
  if (!x || !y || !weight || !bias || !running_mean || !running_var || !save_mean || !save_invstd)
    return fail(B200C_EINVAL, "batch norm res forward: null buffer");
  const bn::FwdArgs a{x, identity, y, nullptr, false, weight, bias, running_mean, running_var,
                      reinterpret_cast<long long*>(num_batches_tracked), save_mean, save_invstd, m, channels, momentum, eps, scratch};
  RT(bn::forward_res(a, noise, rows_per_sample, (cudaStream_t)stream));
  g_launches.fetch_add(2);
  return B200C_OK;
}

// The identity's gradient is dy itself, so the backward takes no identity; the noise check stands in for it.
extern "C" int b200c_bn_backward_res(const void* dy, const void* noise, int rows_per_sample, const void* x, void* g, void* dx,
                                     const float* weight, const float* save_mean, const float* save_invstd, float* grad_weight,
                                     float* grad_bias, int m, int channels, void* scratch, b200c_stream_t stream) {
  int rc = check_bn("batch norm res", 1, m, channels, scratch, 1, nullptr, nullptr, nullptr);
  if (!rc) rc = check_res("batch norm res", m, channels, noise, noise, rows_per_sample);
  if (rc) return rc;
  if (!dy || !x || !dx || !weight || !save_mean || !save_invstd || !grad_weight || !grad_bias || (noise && !g))
    return fail(B200C_EINVAL, "batch norm res backward: null buffer");
  if (g && !noise) return fail(B200C_EINVAL, "batch norm res backward: g without noise (g is dy)");
  const bn::BwdArgs a{dy, nullptr, nullptr, nullptr, x, g, dx, false, weight, save_mean, save_invstd, nullptr, grad_weight, grad_bias,
                      m, channels, scratch};
  RT(bn::backward_res(a, noise, rows_per_sample, (cudaStream_t)stream));
  g_launches.fetch_add(2);
  return B200C_OK;
}

extern "C" int b200c_bn_infer_res(const void* x, const void* identity, void* y, const void* weight, const void* bias,
                                  const void* running_mean, const void* running_var, int param_bf16, float eps, int m, int channels,
                                  b200c_stream_t stream) {
  int rc = check_infer("batch norm infer res", param_bf16, m, channels);
  if (!rc) rc = check_res("batch norm infer res", m, channels, identity, nullptr, 0);
  if (rc) return rc;
  if (!x || !y || !weight || !bias || !running_mean || !running_var) return fail(B200C_EINVAL, "batch norm infer res: null buffer");
  RT(bn::infer_res({x, identity, y, {weight, bias, running_mean, running_var, eps}, {}, false, param_bf16 != 0, m, channels, 0, 0},
                   (cudaStream_t)stream));
  g_launches.fetch_add(1);
  return B200C_OK;
}

// A batch norm and ReLU over a channel concatenation (norm_cat.cuh): the shape (m >= 2 in training: torch's batch norm
// takes more than one value per channel, and the running variance's m / (m - 1) needs it), the segment table, and
// the 16-byte grid of every segment and of the whole-tensor operands `grid`.
static int check_cat(const char* site, int min_m, int m, int c, const void* const* segs, const int* seg_channels, int nsegs,
                     std::initializer_list<const void*> grid) {
  if (m < min_m || c < 1 || c > bn::kMaxChannels || (int64_t)m * c > INT32_MAX) return fail(B200C_EINVAL, "%s: bad shape m=%d c=%d", site, m, c);
  if (nsegs < 1 || nsegs > bn::kMaxCatSegs) return fail(B200C_EINVAL, "%s: nsegs=%d outside 1..%d", site, nsegs, bn::kMaxCatSegs);
  if (!segs || !seg_channels) return fail(B200C_EINVAL, "%s: null segment table", site);
  int64_t total = 0;
  for (int s = 0; s < nsegs; s++) {
    if (!segs[s]) return fail(B200C_EINVAL, "%s: segment %d is null", site, s);
    if (seg_channels[s] < 8 || seg_channels[s] % 8) return fail(B200C_EINVAL, "%s: segment %d has %d channels, not a positive multiple of 8", site, s, seg_channels[s]);
    if (reinterpret_cast<uintptr_t>(segs[s]) % 16) return fail(B200C_EINVAL, "%s: segment %d is off the 16-byte grid", site, s);
    total += seg_channels[s];
  }
  if (total != c) return fail(B200C_EINVAL, "%s: the segments' channels sum to %lld, not channels=%d", site, (long long)total, c);
  for (const void* p : grid)
    if (reinterpret_cast<uintptr_t>(p) % 16) return fail(B200C_EINVAL, "%s: y, dy or dx is off the 16-byte grid", site);
  return B200C_OK;
}

extern "C" int b200c_bn_forward_cat(const void* const* segs, const int* seg_channels, int nsegs, void* y, uint8_t* mask,
                                    const float* weight, const float* bias, float* running_mean, float* running_var,
                                    int64_t* num_batches_tracked, float* save_mean, float* save_invstd, int m, int channels,
                                    float momentum, float eps, void* scratch, b200c_stream_t stream) {
  if (!y || !mask || !weight || !bias || !running_mean || !running_var || !save_mean || !save_invstd || !scratch)
    return fail(B200C_EINVAL, "batch norm cat forward: null buffer");
  int rc = check_cat("batch norm cat", 2, m, channels, segs, seg_channels, nsegs, {y});
  if (rc) return rc;
  const bn::FwdArgs a{nullptr, nullptr, y, mask, true, weight, bias, running_mean, running_var,
                      reinterpret_cast<long long*>(num_batches_tracked), save_mean, save_invstd, m, channels, momentum, eps, scratch};
  RT(bn::forward_cat({segs, seg_channels, nsegs}, a, (cudaStream_t)stream));
  g_launches.fetch_add(2);
  return B200C_OK;
}

extern "C" int b200c_bn_backward_cat(const void* dy, const uint8_t* mask, const void* const* segs, const int* seg_channels, int nsegs,
                                     void* dx, const float* weight, const float* save_mean, const float* save_invstd, float* grad_weight,
                                     float* grad_bias, int m, int channels, void* scratch, b200c_stream_t stream) {
  if (!dy || !mask || !dx || !weight || !save_mean || !save_invstd || !grad_weight || !grad_bias || !scratch)
    return fail(B200C_EINVAL, "batch norm cat backward: null buffer");
  int rc = check_cat("batch norm cat", 2, m, channels, segs, seg_channels, nsegs, {dy, dx});
  if (rc) return rc;
  const bn::BwdArgs a{dy, nullptr, nullptr, mask, nullptr, nullptr, dx, true, weight, save_mean, save_invstd, nullptr, grad_weight,
                      grad_bias, m, channels, scratch};
  RT(bn::backward_cat({segs, seg_channels, nsegs}, a, (cudaStream_t)stream));
  g_launches.fetch_add(2);
  return B200C_OK;
}

extern "C" int b200c_bn_infer_cat(const void* const* segs, const int* seg_channels, int nsegs, void* y, const void* weight,
                                  const void* bias, const void* running_mean, const void* running_var, int param_bf16, float eps, int m,
                                  int channels, b200c_stream_t stream) {
  if (!y || !weight || !bias || !running_mean || !running_var) return fail(B200C_EINVAL, "batch norm infer cat: null buffer");
  int rc = check_infer("batch norm infer cat", param_bf16, m, channels);
  if (!rc) rc = check_cat("batch norm infer cat", 1, m, channels, segs, seg_channels, nsegs, {y});
  if (rc) return rc;
  RT(bn::infer_cat({segs, seg_channels, nsegs}, {nullptr, nullptr, y, {weight, bias, running_mean, running_var, eps}, {}, false,
                                                 param_bf16 != 0, m, channels, 0, 0},
                   (cudaStream_t)stream));
  g_launches.fetch_add(1);
  return B200C_OK;
}

// A batch norm and ReLU whose output is a channel slice of a wider tensor (norm_slice.cuh): the shape (m >= min_m; m * c
// and m * ld below 2^31), c % 8 == 0, the row stride `ld` of y or dy (a multiple of 8, at least c), and the 16-byte
// grid of every bf16 operand `grid`.
static int check_slice(const char* site, int min_m, int m, int c, int ld, std::initializer_list<const void*> grid) {
  if (m < min_m || c < 1 || c > bn::kMaxChannels || (int64_t)m * c > INT32_MAX) return fail(B200C_EINVAL, "%s: bad shape m=%d c=%d", site, m, c);
  if (c % 8) return fail(B200C_EINVAL, "%s: channels=%d is not a multiple of 8", site, c);
  if (ld < c || ld % 8 || (int64_t)m * ld > INT32_MAX)
    return fail(B200C_EINVAL, "%s: row stride %d is not a multiple of 8 of at least channels=%d with m * stride below 2^31", site, ld, c);
  for (const void* p : grid)
    if (reinterpret_cast<uintptr_t>(p) % 16) return fail(B200C_EINVAL, "%s: x, y, dy or dx is off the 16-byte grid", site);
  return B200C_OK;
}

extern "C" int b200c_bn_forward_slice(const void* x, void* y, int ldy, uint8_t* mask, const float* weight, const float* bias,
                                      float* running_mean, float* running_var, int64_t* num_batches_tracked, float* save_mean,
                                      float* save_invstd, int m, int channels, float momentum, float eps, void* scratch,
                                      b200c_stream_t stream) {
  if (!x || !y || !mask || !weight || !bias || !running_mean || !running_var || !save_mean || !save_invstd || !scratch)
    return fail(B200C_EINVAL, "batch norm slice forward: null buffer");
  int rc = check_slice("batch norm slice", 2, m, channels, ldy, {x, y});
  if (rc) return rc;
  const bn::FwdArgs a{x, nullptr, y, mask, true, weight, bias, running_mean, running_var,
                      reinterpret_cast<long long*>(num_batches_tracked), save_mean, save_invstd, m, channels, momentum, eps, scratch};
  RT(bn::forward_slice(a, ldy, (cudaStream_t)stream));
  g_launches.fetch_add(2);
  return B200C_OK;
}

extern "C" int b200c_bn_backward_slice(const void* dy, int lddy, const uint8_t* mask, const void* x, void* dx, const float* weight,
                                       const float* save_mean, const float* save_invstd, float* grad_weight, float* grad_bias, int m,
                                       int channels, void* scratch, b200c_stream_t stream) {
  if (!dy || !mask || !x || !dx || !weight || !save_mean || !save_invstd || !grad_weight || !grad_bias || !scratch)
    return fail(B200C_EINVAL, "batch norm slice backward: null buffer");
  int rc = check_slice("batch norm slice", 2, m, channels, lddy, {dy, x, dx});
  if (rc) return rc;
  const bn::BwdArgs a{dy, nullptr, nullptr, mask, x, nullptr, dx, true, weight, save_mean, save_invstd, nullptr, grad_weight, grad_bias,
                      m, channels, scratch};
  RT(bn::backward_slice(a, lddy, (cudaStream_t)stream));
  g_launches.fetch_add(2);
  return B200C_OK;
}

extern "C" int b200c_bn_infer_slice(const void* x, void* y, int ldy, const void* weight, const void* bias, const void* running_mean,
                                    const void* running_var, int param_bf16, float eps, int m, int channels, b200c_stream_t stream) {
  if (!x || !y || !weight || !bias || !running_mean || !running_var) return fail(B200C_EINVAL, "batch norm infer slice: null buffer");
  int rc = check_infer("batch norm infer slice", param_bf16, m, channels);
  if (!rc) rc = check_slice("batch norm infer slice", 1, m, channels, ldy, {x, y});
  if (rc) return rc;
  RT(bn::infer_slice({x, nullptr, y, {weight, bias, running_mean, running_var, eps}, {}, false, param_bf16 != 0, m, channels, 0, 0}, ldy,
                     (cudaStream_t)stream));
  g_launches.fetch_add(1);
  return B200C_OK;
}

// ShuffleNetV2's block end (norm_shuffle.cuh): the form (exactly one of x1 and u), the shape (n, hw >= 1, m = n * hw
// >= min_m, channels 1..kMaxChannels / 2 since the two-batch-norm form takes the dual scratch, n * 2 * channels * hw
// below 2^31) and x1's sample stride (at least channels * hw, its last element below 2^31).
static int check_shuffle(const char* site, int min_m, const void* x1, int x1_stride, const void* u, int n, int hw, int c) {
  if (!x1 == !u) return fail(B200C_EINVAL, "%s: exactly one of x1 and u must be given", site);
  if (n < 1 || hw < 1 || (int64_t)n * hw < min_m || c < 1 || c > bn::kMaxChannels / 2 || (int64_t)n * 2 * c * hw > INT32_MAX)
    return fail(B200C_EINVAL, "%s: bad shape n=%d hw=%d channels=%d", site, n, hw, c);
  if (x1 && (x1_stride < (int64_t)c * hw || (int64_t)(n - 1) * x1_stride + (int64_t)c * hw > INT32_MAX))
    return fail(B200C_EINVAL, "%s: x1's sample stride %d is below channels * hw or reaches past 2^31 elements", site, x1_stride);
  return B200C_OK;
}

extern "C" size_t b200c_bn_shuffle_mask_bytes(int m, int channels) {
  return m < 1 || channels < 1 || channels > bn::kMaxChannels / 2 || (int64_t)m * channels > INT32_MAX ? 0 : bn::shuffle_mask_bytes(m, channels);
}

extern "C" int b200c_bn_forward_shuffle(const void* x1, int x1_stride, const void* u, uint8_t* mask_u, const float* weight_u,
                                        const float* bias_u, float* running_mean_u, float* running_var_u, int64_t* num_batches_tracked_u,
                                        float* save_mean_u, float* save_invstd_u, float momentum_u, float eps_u, const void* t,
                                        uint8_t* mask, const float* weight, const float* bias, float* running_mean, float* running_var,
                                        int64_t* num_batches_tracked, float* save_mean, float* save_invstd, float momentum, float eps,
                                        void* y, int n, int hw, int channels, void* scratch, b200c_stream_t stream) {
  if (!t || !mask || !weight || !bias || !running_mean || !running_var || !save_mean || !save_invstd || !y || !scratch ||
      (u && (!mask_u || !weight_u || !bias_u || !running_mean_u || !running_var_u || !save_mean_u || !save_invstd_u)))
    return fail(B200C_EINVAL, "batch norm shuffle forward: null buffer");
  int rc = check_shuffle("batch norm shuffle", 2, x1, x1_stride, u, n, hw, channels);
  if (rc) return rc;
  const int m = n * hw;
  const bn::FwdArgs a{t, nullptr, y, mask, true, weight, bias, running_mean, running_var,
                      reinterpret_cast<long long*>(num_batches_tracked), save_mean, save_invstd, m, channels, momentum, eps, scratch};
  const bn::FwdArgs b{u, nullptr, nullptr, mask_u, true, weight_u, bias_u, running_mean_u, running_var_u,
                      reinterpret_cast<long long*>(num_batches_tracked_u), save_mean_u, save_invstd_u, m, channels, momentum_u, eps_u, scratch};
  RT(bn::forward_shuffle(a, u ? &b : nullptr, x1, x1_stride, hw, (cudaStream_t)stream));
  g_launches.fetch_add(2);
  return B200C_OK;
}

// dy is read two channels at a time (4 bytes), so it sits on the 4-byte grid.
extern "C" int b200c_bn_backward_shuffle(const void* dy, const void* u, const uint8_t* mask_u, void* du, const float* weight_u,
                                         const float* save_mean_u, const float* save_invstd_u, float* grad_weight_u, float* grad_bias_u,
                                         const void* t, const uint8_t* mask, void* dt, const float* weight, const float* save_mean,
                                         const float* save_invstd, float* grad_weight, float* grad_bias, int m, int channels,
                                         void* scratch, b200c_stream_t stream) {
  if (!dy || !t || !mask || !dt || !weight || !save_mean || !save_invstd || !grad_weight || !grad_bias || !scratch ||
      (u && (!mask_u || !du || !weight_u || !save_mean_u || !save_invstd_u || !grad_weight_u || !grad_bias_u)))
    return fail(B200C_EINVAL, "batch norm shuffle backward: null buffer");
  if (m < 2 || channels < 1 || channels > bn::kMaxChannels / 2 || (int64_t)m * 2 * channels > INT32_MAX)
    return fail(B200C_EINVAL, "batch norm shuffle: bad shape m=%d channels=%d", m, channels);
  if (reinterpret_cast<uintptr_t>(dy) % 4) return fail(B200C_EINVAL, "batch norm shuffle: dy is off the 4-byte grid");
  const bn::BwdArgs a{dy, nullptr, nullptr, mask, t, nullptr, dt, true, weight, save_mean, save_invstd, nullptr, grad_weight, grad_bias,
                      m, channels, scratch};
  const bn::BwdArgs b{dy, nullptr, nullptr, mask_u, u, nullptr, du, true, weight_u, save_mean_u, save_invstd_u, nullptr, grad_weight_u,
                      grad_bias_u, m, channels, scratch};
  RT(bn::backward_shuffle(a, u ? &b : nullptr, (cudaStream_t)stream));
  g_launches.fetch_add(2);
  return B200C_OK;
}

extern "C" int b200c_bn_infer_shuffle(const void* x1, int x1_stride, const void* u, const void* weight_u, const void* bias_u,
                                      const void* running_mean_u, const void* running_var_u, float eps_u, const void* t,
                                      const void* weight, const void* bias, const void* running_mean, const void* running_var, float eps,
                                      void* y, int param_bf16, int n, int hw, int channels, b200c_stream_t stream) {
  if (!t || !weight || !bias || !running_mean || !running_var || !y || (u && (!weight_u || !bias_u || !running_mean_u || !running_var_u)))
    return fail(B200C_EINVAL, "batch norm infer shuffle: null buffer");
  int rc = check_shuffle("batch norm infer shuffle", 1, x1, x1_stride, u, n, hw, channels);
  if (!rc) rc = check_infer("batch norm infer shuffle", param_bf16, n * hw, channels);
  if (rc) return rc;
  RT(bn::infer_shuffle({t, u, y, {weight, bias, running_mean, running_var, eps}, {weight_u, bias_u, running_mean_u, running_var_u, eps_u},
                        u != nullptr, param_bf16 != 0, n * hw, channels, 0, 0},
                       x1, x1_stride, hw, (cudaStream_t)stream));
  g_launches.fetch_add(1);
  return B200C_OK;
}

// ------------------------------------------------------------------------------------------------
// squeeze-and-excitation (se_kernels.cuh, launched by inst_se.cu): one kernel per call
// ------------------------------------------------------------------------------------------------
// The shape checks of every call.  With one channel and more than one row the reduced dimension is the fastest one,
// where torch's reduction takes another path (vectorize along input), so the reducing kernels reject it.
static int check_se(const char* site, int n, int c, int hw, bool reduce) {
  if (n < 1 || c < 1 || hw < 1 || (int64_t)n * c * hw > INT32_MAX)
    return fail(B200C_EINVAL, "%s: bad shape n=%d c=%d hw=%d", site, n, c, hw);
  if (reduce && c == 1 && hw > 1) return fail(B200C_EINVAL, "%s: one channel with hw=%d reduces along the fastest dimension", site, hw);
  return B200C_OK;
}

extern "C" size_t b200c_se_scratch_bytes(int n, int c, int hw) {
  if (n < 1 || c < 1 || hw < 1 || (int64_t)n * c * hw > INT32_MAX) return 0;
  cudaError_t e;
  size_t bytes = se::scratch_bytes(n, c, hw, &e);
  if (e != cudaSuccess) fail(B200C_ECUDA, "se scratch: %s", cudaGetErrorString(e));
  return bytes;
}

static int check_se_scratch(const char* site, int n, int c, int hw, const void* scratch, size_t scratch_bytes) {
  if (!scratch) return fail(B200C_EINVAL, "%s: null scratch", site);
  const size_t need = b200c_se_scratch_bytes(n, c, hw);
  if (!need) return B200C_ECUDA;
  if (scratch_bytes < need) return fail(B200C_EINVAL, "%s: scratch of %zu bytes, needs %zu", site, scratch_bytes, need);
  return B200C_OK;
}

extern "C" int b200c_se_pool(const void* x, void* pooled, int n, int channels, int hw, void* scratch, size_t scratch_bytes,
                             b200c_stream_t stream) {
  int rc = check_se("se pool", n, channels, hw, true);
  if (!rc && (!x || !pooled)) rc = fail(B200C_EINVAL, "se pool: null buffer");
  if (!rc) rc = check_se_scratch("se pool", n, channels, hw, scratch, scratch_bytes);
  if (rc) return rc;
  RT(se::pool(x, pooled, n, channels, hw, scratch, (cudaStream_t)stream));
  g_launches.fetch_add(1);
  return B200C_OK;
}

extern "C" int b200c_se_scale(const void* x, const void* s, void* y, int n, int channels, int hw, b200c_stream_t stream) {
  int rc = check_se("se scale", n, channels, hw, false);
  if (rc) return rc;
  if (!x || !s || !y) return fail(B200C_EINVAL, "se scale: null buffer");
  RT(se::scale(x, s, y, n, channels, hw, (cudaStream_t)stream));
  g_launches.fetch_add(1);
  return B200C_OK;
}

extern "C" int b200c_se_backward_reduce(const void* dy, const void* x, void* ds, int n, int channels, int hw, void* scratch,
                                        size_t scratch_bytes, b200c_stream_t stream) {
  int rc = check_se("se backward reduce", n, channels, hw, true);
  if (!rc && (!dy || !x || !ds)) rc = fail(B200C_EINVAL, "se backward reduce: null buffer");
  if (!rc) rc = check_se_scratch("se backward reduce", n, channels, hw, scratch, scratch_bytes);
  if (rc) return rc;
  RT(se::backward_reduce(dy, x, ds, n, channels, hw, scratch, (cudaStream_t)stream));
  g_launches.fetch_add(1);
  return B200C_OK;
}

extern "C" int b200c_se_backward_elemt(const void* dy, const void* s, const void* gp, void* dx, int n, int channels, int hw,
                                       b200c_stream_t stream) {
  int rc = check_se("se backward elemt", n, channels, hw, false);
  if (rc) return rc;
  if (!dy || !s || !gp || !dx) return fail(B200C_EINVAL, "se backward elemt: null buffer");
  RT(se::backward_elemt(dy, s, gp, dx, n, channels, hw, (cudaStream_t)stream));
  g_launches.fetch_add(1);
  return B200C_OK;
}

extern "C" int b200c_broadcast(b200c_comm_t* c, void* buf, size_t count, int dtype, int root, b200c_stream_t stream) {
  int rc = check_ready(c);
  if (rc) return rc;
  size_t esz = b200c_dtype_size(dtype);
  if (!esz) return fail(B200C_EINVAL, "bad dtype %d", dtype);
  if (root < 0 || root >= c->world) return fail(B200C_EINVAL, "bad root %d", root);
  if (count == 0 || c->world == 1) return B200C_OK;
  if (!buf) return fail(B200C_EINVAL, "null buffer");
  cudaStream_t s = (cudaStream_t)stream;
  DeviceGuard g(c->device);
  const int W = c->world;
  return run_pieces(c, count * esz, c->cfg.staging_bytes / 16 * 16, "broadcast", [&](CollArgs& a, size_t done, uint32_t& rounds) -> int {
    const size_t n = a.n;
    a.in = static_cast<char*>(buf) + done; a.out = static_cast<char*>(buf) + done;
    a.root = root;
    int grid;
    // every rank takes the same decision from (n, world, multicast)
    const bool mc = c->mc_arena && c->bcast_mc;
    const bool big = c->cfg.bcast_rounds_min_bytes && n >= c->cfg.bcast_rounds_min_bytes;
    const bool mc_rounds = big && mc && W > 2 && n % 16 == 0;     // scatter + multicast allgather
    const bool uc_rounds = big && !mc_rounds && (W == 2 || !mc);  // pipelined unicast push
    if (mc_rounds && (((uintptr_t)a.in) & 15) != 0)
      return fail(B200C_EINVAL, "broadcast of >= %llu bytes needs a 16-byte aligned buffer", (unsigned long long)c->cfg.bcast_rounds_min_bytes);
    if (mc_rounds) {
      a.chunk = round_up((n + W - 1) / W, 16);
      plan_rounds(a.chunk, 1, 16, c->cfg.max_blocks, c->cfg.granule_bytes, &a.tile, &grid, &rounds);
      a.pipe_base = c->pipe_base;
      a.symmetric = 2;
    } else if (uc_rounds) {
      a.chunk = round_up(n, 16);
      plan_rounds(a.chunk, 1, 16, c->cfg.max_blocks, c->cfg.granule_bytes, &a.tile, &grid, &rounds);
      a.pipe_base = c->pipe_base;
      a.symmetric = 3;
    } else {
      a.chunk = round_up(n, 16);
      a.symmetric = (mc && n >= 65536) ? 1 : 0;  // multicast store from the root (same choice on every rank)
      plan_tiles(n, 1, 16, c->cfg.max_blocks, kMinTileBytes, c->cfg.granule_bytes, &a.tile, &grid);
    }
    const bool rounds_mode = mc_rounds || uc_rounds;
    a.sig = make_sig(OPC_BROADCAST, dtype, 0, n, root, a.symmetric);
    if (rounds_mode) k_broadcast_rounds<<<grid, kThreads, 0, s>>>(a);
    else k_broadcast<<<grid, kThreads, 0, s>>>(a);
    return B200C_OK;
  });
}

extern "C" int b200c_barrier(b200c_comm_t* c, b200c_stream_t stream) {
  int rc = check_ready(c);
  if (rc) return rc;
  if (c->world == 1) return B200C_OK;
  DeviceGuard g(c->device);
  return barrier_op(c, (cudaStream_t)stream);
}

// One message over a cell ring: a.buf, a.bytes and the ring's offsets are set by the caller.  *ctr counts the
// cells this side has moved through the ring and only advances once the kernel is really queued.
static int launch_cells(b200c_comm* c, P2PArgs& a, uint32_t* ctr, void (*kernel)(P2PArgs), const char* what, cudaStream_t s) {
  size_t cb = c->cfg.p2p_slot_bytes;
  size_t ncells = (a.bytes + cb - 1) / cb;
  if (ncells > 0x7fffffffull) return fail(B200C_EINVAL, "message too large for the cell ring");
  a.c = c->dev;
  a.first_cell = *ctr; a.ncells = (uint32_t)ncells;
  // no block may wait on a cell that one of its own later iterations has to free: grid <= ring size
  uint32_t grid = (uint32_t)ncells;
  uint32_t lim = c->cfg.max_blocks < (uint32_t)a.cells ? c->cfg.max_blocks : (uint32_t)a.cells;
  if (kernel == k_send) {
    // A sender block publishes `batch` cells per release fence (stride grid).  Small messages keep batch 1
    // (one cell per block: lowest latency); large ones amortise the fence.  All cells of one pass over the
    // grid must fit in the ring together, or a block would wait for an ack that only a later cell of its own
    // pass triggers: grid * batch <= ring cells.
    uint32_t batch = (uint32_t)((ncells + lim - 1) / lim);
    if (batch < 1) batch = 1;
    if (batch > (uint32_t)kSendBatch) batch = kSendBatch;
    a.batch = (int)batch;
    uint32_t lim_s = (uint32_t)a.cells / batch;
    if (lim_s < 1) lim_s = 1;
    if (lim > lim_s) lim = lim_s;
    uint32_t want = ((uint32_t)ncells + batch - 1) / batch;
    grid = want < 1 ? 1 : want;
  }
  if (grid > lim) grid = lim;
  kernel<<<grid, kThreads, 0, s>>>(a);
  int rc = launch_check(c, what);
  if (rc) return rc;
  *ctr += (uint32_t)ncells;
  return B200C_OK;
}
// the pairwise ring of (this rank, peer), or the multi-reader ring of source rank `peer` (`multi`)
static P2PArgs ring_args(b200c_comm* c, void* buf, size_t bytes, int peer, bool multi) {
  P2PArgs a;
  memset(&a, 0, sizeof a);
  a.buf = buf; a.bytes = bytes; a.peer = peer;
  if (multi) { a.off_ring = c->off_mring; a.off_ready = kOffMReady; a.off_ack = kOffMAck; a.cells = (int)c->mcells; }
  else { a.off_ring = c->off_p2p; a.off_ready = kOffP2PReady; a.off_ack = kOffP2PAck; a.cells = (int)c->cfg.p2p_slots; }
  return a;
}

static int p2p_impl(b200c_comm* c, void* buf, size_t bytes, int peer, bool is_send, cudaStream_t s) {
  int rc = check_ready(c);
  if (rc) return rc;
  if (peer < 0 || peer >= c->world) return fail(B200C_EINVAL, "bad peer %d", peer);
  if (peer == c->rank) return fail(B200C_EINVAL, "send/recv to self (rank %d)", peer);
  if (bytes == 0) return B200C_OK;
  if (!buf) return fail(B200C_EINVAL, "null buffer");
  DeviceGuard g(c->device);
  P2PArgs a = ring_args(c, buf, bytes, peer, false);
  if (is_send) return launch_cells(c, a, &c->send_cells[peer], k_send, "send", s);
  return launch_cells(c, a, &c->recv_cells[peer], k_recv, "recv", s);
}
extern "C" int b200c_send(b200c_comm_t* c, const void* buf, size_t bytes, int peer, b200c_stream_t stream) {
  return p2p_impl(c, const_cast<void*>(buf), bytes, peer, true, (cudaStream_t)stream);
}
extern "C" int b200c_recv(b200c_comm_t* c, void* buf, size_t bytes, int peer, b200c_stream_t stream) {
  return p2p_impl(c, buf, bytes, peer, false, (cudaStream_t)stream);
}

extern "C" int b200c_send_multi(b200c_comm_t* c, const void* buf, size_t bytes, const int* peers, int npeers, b200c_stream_t stream) {
  int rc = check_ready(c);
  if (rc) return rc;
  if (!peers || npeers < 1) return fail(B200C_EINVAL, "no readers");
  uint32_t mask = 0;
  for (int i = 0; i < npeers; i++) {
    if (peers[i] < 0 || peers[i] >= c->world) return fail(B200C_EINVAL, "bad peer %d", peers[i]);
    if (peers[i] == c->rank) return fail(B200C_EINVAL, "send to self (rank %d)", peers[i]);
    if (mask & (1u << peers[i])) return fail(B200C_EINVAL, "peer %d listed twice", peers[i]);
    mask |= 1u << peers[i];
  }
  if (npeers == 1 || c->mcells == 0) {   // a single reader is the pairwise ring (the reader calls b200c_recv)
    if (npeers != 1) return fail(B200C_ESTATE, "multi-reader ring unavailable");
    return p2p_impl(c, const_cast<void*>(buf), bytes, peers[0], true, (cudaStream_t)stream);
  }
  if (c->msend_mask && c->msend_mask != mask)
    return fail(B200C_EUNSUPPORTED, "rank %d already multi-sends to reader set 0x%x; a second reader set (0x%x) must use per-reader sends "
                "(ring positions are counted per source, so every reader has to see every message)", c->rank, c->msend_mask, mask);
  if (bytes == 0) return B200C_OK;
  if (!buf) return fail(B200C_EINVAL, "null buffer");
  DeviceGuard g(c->device);
  P2PArgs a = ring_args(c, const_cast<void*>(buf), bytes, -1, true);
  a.reader_mask = mask;
  rc = launch_cells(c, a, &c->msend_cells, k_send_multi, "send_multi", (cudaStream_t)stream);
  if (rc) return rc;
  c->msend_mask = mask;
  return B200C_OK;
}

extern "C" int b200c_recv_multi(b200c_comm_t* c, void* buf, size_t bytes, int src, b200c_stream_t stream) {
  int rc = check_ready(c);
  if (rc) return rc;
  if (src < 0 || src >= c->world || src == c->rank) return fail(B200C_EINVAL, "bad source %d", src);
  if (c->mcells == 0) return p2p_impl(c, buf, bytes, src, false, (cudaStream_t)stream);
  if (bytes == 0) return B200C_OK;
  if (!buf) return fail(B200C_EINVAL, "null buffer");
  DeviceGuard g(c->device);
  P2PArgs a = ring_args(c, buf, bytes, src, true);
  return launch_cells(c, a, &c->mrecv_cells[src], k_recv, "recv_multi", (cudaStream_t)stream);
}
