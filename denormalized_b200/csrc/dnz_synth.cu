// dnz_synth.cu -- counter-based synthetic sensor stream generated directly in device memory
// (SURVEY.md §8d; value distribution of examples/examples/emit_measurements.rs:30-33,45).  Bit-identical to the
// the host generator used by the tests (orc_synth_fill); bench/test infrastructure, not part of the hot path.
#include "dnz_kernels.h"
#include "dnz_window.h"

namespace dnz {

__host__ __device__ __forceinline__ uint64_t splitmix64(uint64_t x) {
  x += 0x9E3779B97F4A7C15ull;
  uint64_t z = x;
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
  return z ^ (z >> 31);
}

__device__ __forceinline__ int dec_digits(uint64_t v) {
  int n = 1;
  while (v >= 10) { v /= 10; n++; }
  return n;
}

// one CTA per batch; 1024-row chunks with a running byte offset.  key_kind: 0 "sensor_<id>", 1 a UUID string per id, 2 Int64
// keys equal to the id (written to `bytes` as int64 values, row i of the stream at index i; `off` is not written)
__global__ void __launch_bounds__(1024) k_synth(int64_t row0, int64_t n_rows, int64_t batch_rows, uint64_t seed, uint64_t groups,
                                               uint64_t rows_per_ms, int64_t t0_ms, int key_kind, uint64_t key_mul, uint64_t key_add, int64_t* ts, double* val,
                                               int32_t* off, uint8_t* bytes, int64_t bytes_stride) {
  const int64_t b = blockIdx.x;
  const int64_t first = b * batch_rows;
  const int64_t n = min(batch_rows, n_rows - first);
  const int64_t off_stride = (batch_rows + 1 + 3) & ~(int64_t)3;
  int32_t* boff = off + b * off_stride;
  uint8_t* bbytes = bytes + b * bytes_stride;
  __shared__ uint32_t wsum[32];
  __shared__ uint32_t running;
  if (threadIdx.x == 0) { running = 0; if (key_kind != 2) boff[0] = 0; }
  __syncthreads();
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int64_t c = 0; c < n; c += blockDim.x) {
    int64_t k = c + threadIdx.x;
    bool live = k < n;
    uint64_t i = (uint64_t)(row0 + first + k);
    uint64_t r = splitmix64(seed ^ i), r2 = splitmix64(r);
    uint64_t key_id = ((r >> 11) % groups) * key_mul + key_add;
    const bool uuid_keys = key_kind == 1, int_keys = key_kind == 2;
    uint32_t len = (live && !int_keys) ? (uuid_keys ? 36u : 7u + (uint32_t)dec_digits(key_id)) : 0u;
    uint32_t inc = len;
    for (int o = 1; o < 32; o <<= 1) { uint32_t x = __shfl_up_sync(0xffffffffu, inc, o); if (lane >= o) inc += x; }
    if (lane == 31) wsum[warp] = inc;
    __syncthreads();
    if (warp == 0) {
      uint32_t x = wsum[lane], y = x;
      for (int o = 1; o < 32; o <<= 1) { uint32_t z = __shfl_up_sync(0xffffffffu, y, o); if (lane >= o) y += z; }
      wsum[lane] = y - x;   // exclusive prefix of the warp totals
    }
    __syncthreads();
    uint32_t base = running + wsum[warp] + (inc - len);
    if (live) {
      ts[first + k] = t0_ms + (int64_t)(i / rows_per_ms);
      val[first + k] = ((double)(r2 >> 11) * 0x1.0p-53) * 115.0;
      uint8_t* p = bbytes + base;
      if (!int_keys) boff[k + 1] = (int32_t)(base + len);
      if (int_keys) {
        reinterpret_cast<int64_t*>(bytes)[first + k] = (int64_t)key_id;
      } else if (uuid_keys) {
        const char hex[] = "0123456789abcdef";
        uint64_t h1 = splitmix64(key_id), h2 = splitmix64(h1);
        int q = 0;
        for (int d = 0; d < 32; d++) {
          uint64_t src = d < 16 ? h1 : h2; int sh = 60 - 4 * (d & 15);
          if (d == 8 || d == 12 || d == 16 || d == 20) p[q++] = '-';
          p[q++] = (uint8_t)hex[(src >> sh) & 15];
        }
      } else {
        p[0] = 's'; p[1] = 'e'; p[2] = 'n'; p[3] = 's'; p[4] = 'o'; p[5] = 'r'; p[6] = '_';
        int nd = (int)len - 7; uint64_t v = key_id;
        for (int d = nd - 1; d >= 0; d--) { p[7 + d] = (uint8_t)('0' + v % 10); v /= 10; }
      }
    }
    __syncthreads();
    // advance the running offset by this chunk's total (last live thread knows it)
    if (live && (k == n - 1 || threadIdx.x == blockDim.x - 1)) running = base + len;
    __syncthreads();
  }
}

cudaError_t launch_synth(int64_t row0, int64_t n_rows, int64_t batch_rows, uint64_t seed, int64_t groups, int64_t rows_per_ms,
                         int64_t t0_ms, int key_kind, int64_t key_mul, int64_t key_add, int64_t* ts, double* val, int32_t* off, uint8_t* bytes,
                         int64_t bytes_stride, cudaStream_t s) {
  if (n_rows <= 0) return cudaSuccess;
  int64_t nb = (n_rows + batch_rows - 1) / batch_rows;
  k_synth<<<(unsigned)nb, 1024, 0, s>>>(row0, n_rows, batch_rows, seed, (uint64_t)groups, (uint64_t)rows_per_ms, t0_ms, key_kind, (uint64_t)key_mul, (uint64_t)key_add, ts, val,
                                       off, bytes, bytes_stride);
  return cudaGetLastError();
}

}  // namespace dnz

// ------------------------------------------------------------------------------------------------
// C API of the generator (include/dnz_gpu.h)
extern "C" {

struct dnz_synth {
  int dev; void* ts; void* val; void* off; void* bytes; int64_t alg_bytes;
};

int32_t dnz_synth_generate(int32_t device, int64_t row0, int64_t n_rows, int64_t batch_rows, uint64_t seed, int64_t groups,
                           int64_t rows_per_ms, int64_t t0_ms, int32_t key_kind, int64_t key_mul, int64_t key_add, dnz_synth** arena,
                           dnz_device_batch* out, int64_t n_batches) {
  if (!arena || !out || n_rows <= 0 || batch_rows <= 0 || groups <= 0 || rows_per_ms <= 0 || key_kind < 0 || key_kind > 2) { g_last_error = "bad synth arguments"; return DNZ_ERR_INVALID; }
  const bool uuid_keys = key_kind == 1, int_keys = key_kind == 2;
  int64_t nb = (n_rows + batch_rows - 1) / batch_rows;
  if (n_batches < nb) { g_last_error = "batch array too small"; return DNZ_ERR_INVALID; }
  if (cudaSetDevice(device) != cudaSuccess) { g_last_error = "no such CUDA device"; return DNZ_ERR_CUDA; }
  int maxlen = 36;
  if (key_mul < 1) key_mul = 1;
  if (!uuid_keys) { maxlen = 8; for (int64_t v = (groups - 1) * key_mul + key_add; v >= 10; v /= 10) maxlen++; }
  int64_t off_stride = int_keys ? 0 : (batch_rows + 1 + 3) & ~(int64_t)3;
  int64_t bytes_stride = int_keys ? batch_rows * 8 : (batch_rows * maxlen + 15 + 16) & ~(int64_t)15;
  dnz_synth* a = new dnz_synth{device, nullptr, nullptr, nullptr, nullptr, 0};
  auto bail = [&](const char* m) { g_last_error = m; dnz_synth_free(a); return DNZ_ERR_CUDA; };
  if (cudaMalloc(&a->ts, (size_t)n_rows * 8 + 64) != cudaSuccess) return bail("cudaMalloc(ts) failed");
  if (cudaMalloc(&a->val, (size_t)n_rows * 8 + 64) != cudaSuccess) return bail("cudaMalloc(val) failed");
  if (cudaMalloc(&a->off, (size_t)nb * off_stride * 4 + 64) != cudaSuccess) return bail("cudaMalloc(off) failed");
  if (cudaMalloc(&a->bytes, (size_t)nb * bytes_stride + 64) != cudaSuccess) return bail("cudaMalloc(bytes) failed");
  if (launch_synth(row0, n_rows, batch_rows, seed, groups, rows_per_ms, t0_ms, key_kind, key_mul, key_add, (int64_t*)a->ts, (double*)a->val,
                   (int32_t*)a->off, (uint8_t*)a->bytes, bytes_stride, nullptr) != cudaSuccess) return bail("synth launch failed");
  if (cudaDeviceSynchronize() != cudaSuccess) return bail("synth kernel failed");
  // algorithmic bytes: 20 B/row + key bytes (last offset of every batch); Int64 keys: 24 B/row
  std::vector<int32_t> last((size_t)nb, 0);
  for (int64_t b = 0; b < nb && !int_keys; b++) {
    int64_t n = std::min(batch_rows, n_rows - b * batch_rows);
    if (cudaMemcpy(&last[(size_t)b], (int32_t*)a->off + b * off_stride + n, 4, cudaMemcpyDeviceToHost) != cudaSuccess) return bail("memcpy failed");
  }
  a->alg_bytes = (int_keys ? 24 : 20) * n_rows;
  for (int64_t b = 0; b < nb; b++) {
    int64_t n = std::min(batch_rows, n_rows - b * batch_rows);
    a->alg_bytes += last[(size_t)b];
    dnz_device_batch& d = out[b];
    memset(&d, 0, sizeof d);
    d.n_rows = n; d.ts = (int64_t*)a->ts + b * batch_rows; d.val = (double*)a->val + b * batch_rows;
    d.key_off = int_keys ? nullptr : (int32_t*)a->off + b * off_stride; d.key_bytes = (uint8_t*)a->bytes + b * bytes_stride;
  }
  *arena = a;
  return DNZ_OK;
}
int64_t dnz_synth_bytes(const dnz_synth* a) { return a ? a->alg_bytes : 0; }
void dnz_synth_free(dnz_synth* a) {
  if (!a) return;
  cudaSetDevice(a->dev);
  cudaFree(a->ts); cudaFree(a->val); cudaFree(a->off); cudaFree(a->bytes);
  delete a;
}

}  // extern "C"
