// Host-side interface between the C-ABI (b200coll.cu) and the squeeze-and-excitation launchers (inst_se.cu).
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>

namespace b200c {
namespace se {

// Scratch of a site of n samples, c channels and hw rows per sample on the current device: the semaphore region
// (left at zero by every call) and the staging of either reducing kernel.  0 if the shape is out of range.
size_t scratch_bytes(int n, int c, int hw, cudaError_t* err);

// One kernel each.  x, y, dy, dx: bf16 [n][hw][c]; pooled, s, ds, gp: bf16 [n][c].  The reducing calls take the
// scratch (at least scratch_bytes(n, c, hw), zero-filled before its first use) and return cudaErrorInvalidValue if the
// device would split a reduction over more blocks in x than the semaphore region holds.
cudaError_t pool(const void* x, void* pooled, int n, int c, int hw, void* scratch, cudaStream_t s);
cudaError_t scale(const void* x, const void* sc, void* y, int n, int c, int hw, cudaStream_t s);
cudaError_t backward_reduce(const void* dy, const void* x, void* ds, int n, int c, int hw, void* scratch, cudaStream_t s);
cudaError_t backward_elemt(const void* dy, const void* sc, const void* gp, void* dx, int n, int c, int hw, cudaStream_t s);

}  // namespace se
}  // namespace b200c
