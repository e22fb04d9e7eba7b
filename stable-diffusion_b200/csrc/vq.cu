// Vector quantizer of the VQ first stages (taming's VectorQuantizer2.forward, legacy, no remap): nearest codebook entry
// by d = sum(z^2) + sum(e^2) - 2 z.e, lowest index on ties, and the straight-through output z + (e - z).
// One thread per latent pixel; the codebook streams through shared memory in chunks, so its size is not bounded by
// shared memory (8192 x 3 for vq-f4, 16384 x 4 for vq-f8). The decode spends milliseconds in its convolutions; this
// kernel is a small share of it and is kept simple.
#include "../../include/sdb200.h"
#include "host.h"

namespace sdb {

constexpr int VQ_MAX_DIM = 8;
constexpr int VQ_THREADS = 256;
constexpr int VQ_CHUNK = 1024;   // codes per shared-memory chunk: 1024 x (8 + 1) floats = 36 KiB

template <int D>
__global__ void __launch_bounds__(VQ_THREADS) vq_quantize_kernel(const float* __restrict__ z, long long m, float scale,
                                                                 const float* __restrict__ codebook,
                                                                 const float* __restrict__ code_sq, int n_e,
                                                                 float* __restrict__ z_q, long long* __restrict__ indices) {
  __shared__ float es[VQ_CHUNK * D];
  __shared__ float esq[VQ_CHUNK];
  const long long row = blockIdx.x * static_cast<long long>(VQ_THREADS) + threadIdx.x;
  const bool live = row < m;
  float zv[D];
  float zz = 0.f;
#pragma unroll
  for (int k = 0; k < D; ++k) {
    zv[k] = live ? __fmul_rn(scale, z[row * D + k]) : 0.f;
    zz = __fadd_rn(zz, __fmul_rn(zv[k], zv[k]));
  }
  float best = 0.f;
  int best_i = -1;
  for (int c0 = 0; c0 < n_e; c0 += VQ_CHUNK) {
    const int nc = min(VQ_CHUNK, n_e - c0);
    __syncthreads();
    for (int i = threadIdx.x; i < nc * D; i += VQ_THREADS) es[i] = codebook[static_cast<long long>(c0) * D + i];
    for (int i = threadIdx.x; i < nc; i += VQ_THREADS) esq[i] = code_sq[c0 + i];
    __syncthreads();
    for (int j = 0; j < nc; ++j) {
      float dot = 0.f;
#pragma unroll
      for (int k = 0; k < D; ++k) dot = __fmaf_rn(zv[k], es[j * D + k], dot);
      const float d = __fsub_rn(__fadd_rn(zz, esq[j]), __fmul_rn(2.f, dot));
      if (best_i < 0 || d < best) {   // strict: the lowest index wins a tie, as torch.argmin
        best = d;
        best_i = c0 + j;
      }
    }
  }
  if (!live) return;
#pragma unroll
  for (int k = 0; k < D; ++k) {
    const float e = codebook[static_cast<long long>(best_i) * D + k];
    z_q[row * D + k] = __fadd_rn(zv[k], __fsub_rn(e, zv[k]));   // z + (z_q - z).detach(), rounded as the reference
  }
  if (indices) indices[row] = best_i;
}

template <int D>
static void launch_vq(const float* z, long long m, float scale, const float* codebook, const float* code_sq, int n_e,
                      float* z_q, long long* idx, cudaStream_t st) {
  const unsigned blocks = static_cast<unsigned>((m + VQ_THREADS - 1) / VQ_THREADS);
  vq_quantize_kernel<D><<<blocks, VQ_THREADS, 0, st>>>(z, m, scale, codebook, code_sq, n_e, z_q, idx);
}

}  // namespace sdb

using namespace sdb;

extern "C" int sdb_vq_quantize(const float* z, int64_t m, int32_t e_dim, float scale, const float* codebook,
                               const float* code_sq, int32_t n_e, float* z_q, int64_t* indices, sdb_stream_t stream) {
  SDB_REC(sdb_vq_quantize(z, m, e_dim, scale, codebook, code_sq, n_e, z_q, indices, s_));
  SDB_CHECK(z && codebook && code_sq && z_q && m > 0 && n_e > 0, "sdb_vq_quantize: bad arguments");
  SDB_CHECK(e_dim >= 1 && e_dim <= VQ_MAX_DIM, "sdb_vq_quantize: e_dim %d not supported (1 .. %d)", e_dim, VQ_MAX_DIM);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  long long* idx = reinterpret_cast<long long*>(indices);
  switch (e_dim) {
    case 1: launch_vq<1>(z, m, scale, codebook, code_sq, n_e, z_q, idx, st); break;
    case 2: launch_vq<2>(z, m, scale, codebook, code_sq, n_e, z_q, idx, st); break;
    case 3: launch_vq<3>(z, m, scale, codebook, code_sq, n_e, z_q, idx, st); break;
    case 4: launch_vq<4>(z, m, scale, codebook, code_sq, n_e, z_q, idx, st); break;
    case 5: launch_vq<5>(z, m, scale, codebook, code_sq, n_e, z_q, idx, st); break;
    case 6: launch_vq<6>(z, m, scale, codebook, code_sq, n_e, z_q, idx, st); break;
    case 7: launch_vq<7>(z, m, scale, codebook, code_sq, n_e, z_q, idx, st); break;
    default: launch_vq<8>(z, m, scale, codebook, code_sq, n_e, z_q, idx, st); break;
  }
  SDB_LAUNCH_CHECK();
  return 0;
}
