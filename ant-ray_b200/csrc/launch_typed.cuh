// Per-dtype launch tables.  Each inst_<dtype>.cu instantiates this for one storage type so the
// translation units compile in parallel.
#pragma once
#include <type_traits>

#include "coll_kernels.cuh"

namespace b200c {

// The reducing kernels exist once per world size 2 / 4 / 8 and once for the other sizes (WT = 0):
// calls f(std::integral_constant<int, WT>) for the communicator's world size.
template <typename F>
static auto with_world_t(int world, F&& f) {
  switch (world) {
    case 2: return f(std::integral_constant<int, 2>{});
    case 4: return f(std::integral_constant<int, 4>{});
    case 8: return f(std::integral_constant<int, 8>{});
    default: return f(std::integral_constant<int, 0>{});
  }
}

// KIND_LOAD launches nothing: it loads the kernels of every kind for (T, OP, WT) into the context (load_kernels)
enum Kind { KIND_ONESHOT = 0, KIND_TWOSHOT = 1, KIND_REDUCESCATTER = 2, KIND_REDUCE = 3, KIND_LL = 4, KIND_LOAD = 5 };

// cudaFuncGetAttributes loads a kernel that lazy module loading has not loaded yet
template <typename K>
static int load_kernel(K* kernel) {
  cudaFuncAttributes attr;
  return cudaFuncGetAttributes(&attr, kernel) == cudaSuccess ? B200C_OK : B200C_ECUDA;
}

template <typename T, int OP, int WT>
static int launch_kind_w(int kind, const CollArgs& a, int grid, cudaStream_t s) {
  switch (kind) {
    case KIND_LOAD: {
      int rc = load_kernel(k_allreduce_oneshot<T, T, OP, WT>);
      if (!rc) rc = load_kernel(k_allreduce_twoshot<T, T, OP, WT>);
      if (!rc) rc = load_kernel(k_reducescatter<T, OP, WT>);
      if (!rc) rc = load_kernel(k_reduce<T, OP, WT>);
      if (!rc) rc = load_kernel(k_allreduce_ll<T, OP, WT>);
      return rc;
    }
    case KIND_ONESHOT: k_allreduce_oneshot<T, T, OP, WT><<<grid, kThreads, 0, s>>>(a); break;
    case KIND_TWOSHOT: k_allreduce_twoshot<T, T, OP, WT><<<grid, kThreads, 0, s>>>(a); break;
    case KIND_REDUCESCATTER: k_reducescatter<T, OP, WT><<<grid, kThreads, 0, s>>>(a); break;
    case KIND_REDUCE: k_reduce<T, OP, WT><<<grid, kThreads, 0, s>>>(a); break;
    case KIND_LL: k_allreduce_ll<T, OP, WT><<<grid, kLLThreads, 0, s>>>(a); break;
    default: return B200C_EINVAL;
  }
  return B200C_OK;
}

template <typename T, int OP>
static int launch_kind(int kind, const CollArgs& a, int grid, cudaStream_t s) {
  return with_world_t(a.c.world, [&](auto wt) { return launch_kind_w<T, OP, decltype(wt)::value>(kind, a, grid, s); });
}

template <typename T>
static int launch_typed_impl(int kind, int op, const CollArgs& a, int grid, cudaStream_t s) {
  switch (op) {
    case B200C_SUM: case B200C_AVG: return launch_kind<T, B200C_SUM>(kind, a, grid, s);
    case B200C_PROD: return launch_kind<T, B200C_PROD>(kind, a, grid, s);
    case B200C_MAX: return launch_kind<T, B200C_MAX>(kind, a, grid, s);
    case B200C_MIN: return launch_kind<T, B200C_MIN>(kind, a, grid, s);
    default: return B200C_EINVAL;
  }
}

#define B200C_DECLARE_TYPED(name) int launch_##name(int kind, int op, const CollArgs& a, int grid, cudaStream_t s)
B200C_DECLARE_TYPED(i8);
B200C_DECLARE_TYPED(u8);
B200C_DECLARE_TYPED(i32);
B200C_DECLARE_TYPED(u32);
B200C_DECLARE_TYPED(i64);
B200C_DECLARE_TYPED(u64);
B200C_DECLARE_TYPED(f16);
B200C_DECLARE_TYPED(f32);
B200C_DECLARE_TYPED(f64);
B200C_DECLARE_TYPED(bf16);

}  // namespace b200c
