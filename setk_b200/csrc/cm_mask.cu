// cm_mask.cu -- Kaldi CompressedMatrix ("CM": per-column headers + one byte per element) -> the
// float32 [B][T][F] mask batch of the beamformer, on the device.
//
// Replaces (scripts/sptk): kaldi_io.py:248-281 uncompress() as reached from
// apply_adaptive_beamformer.py:139-142 (ScriptReader -> read_compress_mat) when the masks of
// `--mask-format kaldi` were written compressed -- Kaldi's default for feature-like archives.
// A mask row is then 1 byte per TF cell instead of 4: the batched feeder ships the archive's bytes
// as they are (a quarter of the mask traffic over PCIe) and this kernel expands them next to the
// kernels that consume them.
//
// Layout of one matrix, exactly as it lies in an archive behind the "CM " token:
//   { float min_value, float range, int32 num_rows, int32 num_cols }            16 bytes
//   num_cols x { uint16 percentile_0, _25, _75, _100 }                          8 bytes each
//   num_cols x num_rows x uint8                                                 column major
// value(b, col) = piecewise linear between the column's percentiles (kaldi_io.py:266-281), every
// operation a float32 operation in the reference's order (numpy float32 arrays x weak python
// scalars): no FMA contraction, IEEE division -- the result is bit-identical to the reference's.
#include "common.cuh"
#include "launchers.cuh"

namespace setk {

__device__ __forceinline__ float cm_percentile(unsigned short u, float range, float minv) {
  return __fadd_rn(__fdiv_rn(__fmul_rn((float)u, range), 65535.0f), minv);
}
__device__ __forceinline__ float cm_value(int b, float p0, float p1, float p2, float p3) {
  const float fb = (float)b;
  if (b <= 64) return __fadd_rn(__fdiv_rn(__fmul_rn(fb, __fsub_rn(p1, p0)), 64.0f), p0);
  if (b >= 193) return __fadd_rn(__fdiv_rn(__fmul_rn(__fsub_rn(fb, 192.0f), __fsub_rn(p3, p2)), 63.0f), p2);
  return __fadd_rn(__fdiv_rn(__fmul_rn(__fsub_rn(fb, 64.0f), __fsub_rn(p2, p1)), 128.0f), p1);
}

// block (32, 8): a tile of 32 rows (t) x 32 columns (f); bytes are read along t (contiguous in the
// column-major archive), floats written along f (contiguous in [T][F])
__global__ void cm_masks_kernel(const unsigned char* blobs, long long slot_bytes, int T, int F, float* out,
                                int* status) {
  __shared__ float tile[32][33];
  __shared__ float pct[32][4];
  const int b = blockIdx.z;
  const unsigned char* blob = blobs + (long long)b * slot_bytes;
  const float minv = *reinterpret_cast<const float*>(blob);
  const float range = *reinterpret_cast<const float*>(blob + 4);
  const int rows = *reinterpret_cast<const int*>(blob + 8);
  const int cols = *reinterpret_cast<const int*>(blob + 12);
  const bool ok = cols == F && rows >= 0 && rows <= T && 16 + (long long)cols * (8 + rows) <= slot_bytes;
  const int t0 = blockIdx.x * 32, f0 = blockIdx.y * 32;
  const int tx = threadIdx.x, ty = threadIdx.y;
  if (!ok) {
    if (blockIdx.x == 0 && blockIdx.y == 0 && tx == 0 && ty == 0) status[b] = 1;
    for (int i = ty; i < 32; i += 8)
      if (t0 + i < T && f0 + tx < F) out[((long long)b * T + t0 + i) * F + f0 + tx] = 0.f;
    return;
  }
  if (ty < 4 && f0 + tx < F) {
    const unsigned short u = *reinterpret_cast<const unsigned short*>(blob + 16 + (long long)(f0 + tx) * 8 + 2 * ty);
    pct[tx][ty] = cm_percentile(u, range, minv);
  }
  __syncthreads();
  const unsigned char* data = blob + 16 + (long long)cols * 8;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int fl = ty + 8 * i, f = f0 + fl, t = t0 + tx;
    float v = 0.f;
    if (f < F && t < rows) v = cm_value(data[(long long)f * rows + t], pct[fl][0], pct[fl][1], pct[fl][2], pct[fl][3]);
    tile[fl][tx] = v;
  }
  __syncthreads();
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int tl = ty + 8 * i, t = t0 + tl, f = f0 + tx;
    if (t < T && f < F) out[((long long)b * T + t) * F + f] = tile[tx][tl];
  }
}

cudaError_t run_cm_masks(const unsigned char* blobs, long long slot_bytes, int B, int T, int F, float* out,
                         int* status, void* stream) {
  if (B == 0 || T == 0 || F == 0) return cudaSuccess;
  const dim3 grid((unsigned)((T + 31) / 32), (unsigned)((F + 31) / 32), (unsigned)B);
  return launch(cm_masks_kernel, grid, dim3(32, 8), 0, stream, false, blobs, slot_bytes, T, F, out, status);
}

}  // namespace setk
