// scatter_bench.cu -- microbenchmark behind the k_aggregate redesign (round 1).
// Question: what does one scattered 32 B-sector transaction cost on the GPU at hand, by kind, and can the four per-row
// reductions {count, sum, min, max} be issued in fewer L1tex wavefronts?
//   build: nvcc -O3 -std=c++17 -gencode arch=compute_90a,code=sm_90a -o scatter_bench scatter_bench.cu
//   run:   ./scatter_bench [rows_log2=26] [groups=100000]
// Every variant processes `rows` synthetic rows (gid = splitmix(i) % G, v = uniform) against a G x 32 B state table
// and (when probing) a dictionary sized as the operator sizes it (dict_slots_per_group: gcap x 16 slots of 32 B up to 1 Mi
// groups, gcap = G rounded up to a power of two; 2 Mi slots = 64 MiB for cfg 2's 100 K groups), of which G slots are
// occupied, so the access pattern and the L2 line footprint equal cfg 2's.
#include <cstdio>
#include <cstdlib>
#include <cstdint>
#include <cuda_runtime.h>

#define CK(x) do { cudaError_t e = (x); if (e != cudaSuccess) { printf("CUDA error %s at %d\n", cudaGetErrorString(e), __LINE__); exit(1); } } while (0)

struct __align__(32) State { double cnt; double sum; unsigned long long mnk; unsigned long long mxk; };
struct __align__(32) Slot { uint64_t a, b, c, d; };

__device__ __forceinline__ uint64_t splitmix(uint64_t x) {
  x += 0x9E3779B97F4A7C15ull; x = (x ^ (x >> 30)) * 0xBF58476D1CE4E5B9ull; x = (x ^ (x >> 27)) * 0x94D049BB133111EBull; return x ^ (x >> 31);
}
__device__ __forceinline__ void red_add_u64(void* p, unsigned long long v) { asm volatile("red.global.add.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory"); }
__device__ __forceinline__ void red_add_f64(void* p, double v) { asm volatile("red.global.add.f64 [%0], %1;" ::"l"(p), "d"(v) : "memory"); }
__device__ __forceinline__ void red_max_u64(void* p, unsigned long long v) { asm volatile("red.global.max.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory"); }
__device__ __forceinline__ void ld_slot(const Slot* p, uint64_t& a, uint64_t& b, uint64_t& c, uint64_t& d) {
  // two 16 B loads of the 32 B slot: sm_90 has no 256-bit load
  asm volatile("ld.relaxed.gpu.global.v2.u64 {%0,%1}, [%2];" : "=l"(c), "=l"(d) : "l"(reinterpret_cast<const char*>(p) + 16) : "memory");
  asm volatile("ld.relaxed.gpu.global.v2.u64 {%0,%1}, [%2];" : "=l"(a), "=l"(b) : "l"(p) : "memory");
}
__device__ __forceinline__ void ld_slot_nc(const Slot* p, uint64_t& a, uint64_t& b, uint64_t& c, uint64_t& d) {
  asm volatile("ld.global.nc.v2.u64 {%0,%1}, [%2];" : "=l"(c), "=l"(d) : "l"(reinterpret_cast<const char*>(p) + 16) : "memory");
  asm volatile("ld.global.nc.v2.u64 {%0,%1}, [%2];" : "=l"(a), "=l"(b) : "l"(p) : "memory");
}
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

enum Variant { V_RED4 = 0, V_RED2, V_PAIR, V_PAIR_ADD, V_PROBE, V_PROBE_NC, V_PROBE_RED4, V_PROBE_PAIR, V_PROBE_HINT, V_PROBE_HINT_SCALAR,
               V_BULK, V_QUAD_ADD, V_RED1, V_PROBE_RED1, V_PROBE16, V_TEX32, V_TEX16, V_TEX32_HINT, V_PROBE_HINT_XOR, V_XOR_ADD,
               V_PROBE_PAIRED, V_PROBE_PAIRED_HINT_XOR, V_COUNT };
static const char* NAMES[] = {"red4 (cnt,sum,min,max scalar REDs)", "red2 (cnt,sum scalar)", "pair (add.f64 x2 lanes + max.u64 x2 lanes, 16 rows/instr)",
                              "pair_add only", "probe only (ld.relaxed.gpu 2 x v2.u64)", "probe only (ld.global.nc 2 x v2.u64)", "probe + red4  [= round-1 kernel]",
                              "probe + pair", "probe + pair_add + 6% pair_max (hint)", "probe + red2 + 6% red max x2 (hint, scalar)",
                              "cp.reduce.async.bulk 16 B add.f64 + 16 B max.u64", "quad add.f64 (4 lanes/sector, 8 rows/instr)", "red1 (one scalar RED)",
                              "probe + red1", "probe only 16 B (v2.u64)", "TEX probe 32 B (2 x tex1Dfetch<uint4>)", "TEX probe 16 B (1 x tex1Dfetch<uint4>)",
                              "TEX probe 32 B + xor-pair add + 6% own-lane max", "LDG probe + xor-pair add + 6% own-lane max", "xor-pair add only (1 shuffle)",
                              "lane-paired probe only (2 lanes x 16 B per slot, 16 rows/instr)", "lane-paired probe + xor-pair add + 6% own-lane max"};

template <int V>
__global__ void __launch_bounds__(512) k_bench(State* __restrict__ st, const Slot* __restrict__ dict, uint32_t mask, uint64_t rows, uint32_t G,
                                               unsigned long long* sink, cudaTextureObject_t tex) {
  const int lane = threadIdx.x & 31;
  uint64_t acc = 0;
  __shared__ __align__(16) unsigned long long stage[512 * 4];
  for (uint64_t base = (uint64_t)blockIdx.x * blockDim.x; base < rows; base += (uint64_t)gridDim.x * blockDim.x) {
    uint64_t i = base + threadIdx.x;
    uint64_t r = splitmix(i);
    uint32_t gid = (uint32_t)((r >> 11) % G);
    double v = (double)(splitmix(r) >> 11) * (115.0 / 9007199254740992.0);
    unsigned long long o = (unsigned long long)__double_as_longlong(v) | 0x8000000000000000ull;
    unsigned long long mnk = 0xFFEFFFFFFFFFFFFFull - o, mxk = o - 0x0010000000000000ull;
    bool hint_pass = true;
    if (V == V_PROBE || V == V_PROBE_NC || V == V_PROBE_RED4 || V == V_PROBE_PAIR || V == V_PROBE_HINT || V == V_PROBE_HINT_SCALAR || V == V_PROBE_RED1) {
      uint32_t idx = (uint32_t)splitmix(gid) & mask;
      uint64_t a, b, c, d;
      if (V == V_PROBE_NC) ld_slot_nc(dict + idx, a, b, c, d); else ld_slot(dict + idx, a, b, c, d);
      acc += a ^ b ^ c ^ d;
      gid = (uint32_t)((gid + (a & 1)) % G);     // make the updates depend on the probe (a is 0)
      hint_pass = ((r >> 40) & 1023) < 61;       // ~6 % of the rows beat the hint
    }
    if (V == V_PROBE_PAIRED || V == V_PROBE_PAIRED_HINT_XOR) {
      // k_aggregate's probe (ld_slot_paired): lanes 2j / 2j+1 load the two halves of the even lane's slot, then of the odd
      // lane's slot; one xor-shuffle of 16 B hands each lane the half its partner loaded
      const uint32_t idx = (uint32_t)splitmix(gid) & mask, idx2 = __shfl_xor_sync(0xffffffffu, idx, 1), odd = lane & 1;
      const char* base = reinterpret_cast<const char*>(dict);
      uint64_t x0, x1, y0, y1;
      asm volatile("ld.relaxed.gpu.global.v2.u64 {%0,%1}, [%2];" : "=l"(x0), "=l"(x1) : "l"(base + (size_t)(odd ? idx2 : idx) * 32 + 16 * odd) : "memory");
      asm volatile("ld.relaxed.gpu.global.v2.u64 {%0,%1}, [%2];" : "=l"(y0), "=l"(y1) : "l"(base + (size_t)(odd ? idx : idx2) * 32 + 16 * (odd ^ 1)) : "memory");
      const uint64_t c = __shfl_xor_sync(0xffffffffu, odd ? x0 : y0, 1), d = __shfl_xor_sync(0xffffffffu, odd ? x1 : y1, 1);
      const uint64_t a = odd ? y0 : x0, b = odd ? y1 : x1;
      acc += a ^ b ^ c ^ d;
      gid = (uint32_t)((gid + (a & 1)) % G);
      hint_pass = ((r >> 40) & 1023) < 61;
    }
    if (V == V_PROBE16) {
      uint32_t idx = (uint32_t)splitmix(gid) & mask; uint64_t a, b;
      asm volatile("ld.relaxed.gpu.global.v2.u64 {%0,%1}, [%2];" : "=l"(a), "=l"(b) : "l"(dict + idx) : "memory");
      acc += a ^ b;
    }

    if (V == V_TEX32 || V == V_TEX16 || V == V_TEX32_HINT) {
      uint32_t idx = (uint32_t)splitmix(gid) & mask;
      uint4 a = tex1Dfetch<uint4>(tex, (int)(2u * idx));
      acc += a.x ^ a.y ^ a.z ^ a.w;
      if (V != V_TEX16) { uint4 b = tex1Dfetch<uint4>(tex, (int)(2u * idx + 1u)); acc += b.x ^ b.y ^ b.z ^ b.w; gid = (uint32_t)((gid + (b.x & 1)) % G); }
      else gid = (uint32_t)((gid + (a.x & 1)) % G);
      hint_pass = ((r >> 40) & 1023) < 61;
    }
    if (V == V_PROBE_HINT_XOR) {
      uint32_t idx = (uint32_t)splitmix(gid) & mask;
      uint64_t a, b, c, d; ld_slot(dict + idx, a, b, c, d);
      acc += a ^ b ^ c ^ d; gid = (uint32_t)((gid + (a & 1)) % G); hint_pass = ((r >> 40) & 1023) < 61;
    }
    if (V == V_TEX32_HINT || V == V_PROBE_HINT_XOR || V == V_XOR_ADD || V == V_PROBE_PAIRED_HINT_XOR) {
      // lanes 2j / 2j+1 share one sector per instruction; ONE xor-shuffle of the group id serves both halves:
      // half 0 = rows of even lanes (own lane adds the sum, the partner adds the count), half 1 = rows of odd lanes
      const uint32_t g2 = __shfl_xor_sync(0xffffffffu, gid, 1);
      const int odd = lane & 1;
#pragma unroll
      for (int half = 0; half < 2; half++) {
        const bool own = (odd == half);
        State* s2 = st + (own ? gid : g2);
        red_add_f64(reinterpret_cast<double*>(s2) + (own ? 1 : 0), own ? v : 1.0);
      }
      if (V != V_XOR_ADD && hint_pass) { red_max_u64(&st[gid].mnk, mnk); }
    }
    State* s = st + gid;
    if (V == V_RED4 || V == V_PROBE_RED4) { red_add_u64(&s->cnt, 1ull); red_add_f64(&s->sum, v); red_max_u64(&s->mnk, mnk); red_max_u64(&s->mxk, mxk); }
    if (V == V_RED2) { red_add_u64(&s->cnt, 1ull); red_add_f64(&s->sum, v); }
    if (V == V_RED1 || V == V_PROBE_RED1) { red_add_f64(&s->sum, v); }
    if (V == V_PROBE_HINT_SCALAR) {
      red_add_u64(&s->cnt, 1ull); red_add_f64(&s->sum, v);
      if (hint_pass) { red_max_u64(&s->mnk, mnk); red_max_u64(&s->mxk, mxk); }
    }
    if (V == V_PAIR || V == V_PAIR_ADD || V == V_PROBE_PAIR || V == V_PROBE_HINT) {
      // lane L serves field (L & 1) of the row held by lane (L >> 1) + 16 * half
#pragma unroll
      for (int half = 0; half < 2; half++) {
        int src = (lane >> 1) + 16 * half;
        uint32_t g2 = __shfl_sync(0xffffffffu, gid, src);
        double v2 = __shfl_sync(0xffffffffu, v, src);
        State* s2 = st + g2;
        red_add_f64(reinterpret_cast<double*>(s2) + (lane & 1), (lane & 1) ? v2 : 1.0);
        if (V == V_PAIR || V == V_PROBE_PAIR) {
          unsigned long long k2 = __shfl_sync(0xffffffffu, (lane & 1) ? mxk : mnk, src);   // wrong field for odd/even mix: fine for timing
          red_max_u64(reinterpret_cast<unsigned long long*>(s2) + 2 + (lane & 1), k2);
        }
        if (V == V_PROBE_HINT) {
          bool hp = __shfl_sync(0xffffffffu, hint_pass, src);
          unsigned long long k2 = __shfl_sync(0xffffffffu, mnk, src);
          if (hp) red_max_u64(reinterpret_cast<unsigned long long*>(s2) + 2 + (lane & 1), k2);
        }
      }
    }
    if (V == V_QUAD_ADD) {
#pragma unroll
      for (int q = 0; q < 4; q++) {
        int src = (lane >> 2) + 8 * q;
        uint32_t g2 = __shfl_sync(0xffffffffu, gid, src);
        double v2 = __shfl_sync(0xffffffffu, v, src);
        red_add_f64(reinterpret_cast<double*>(st + g2) + (lane & 3), v2);
      }
    }
    if (V == V_BULK) {
      unsigned long long* my = stage + threadIdx.x * 4;
      my[0] = (unsigned long long)__double_as_longlong(1.0); my[1] = (unsigned long long)__double_as_longlong(v); my[2] = mnk; my[3] = mxk;
      asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
      asm volatile("cp.reduce.async.bulk.global.shared::cta.bulk_group.add.f64 [%0], [%1], 16;" ::"l"(&s->cnt), "r"(smem_u32(my)) : "memory");
      asm volatile("cp.reduce.async.bulk.global.shared::cta.bulk_group.max.u64 [%0], [%1], 16;" ::"l"(&s->mnk), "r"(smem_u32(my + 2)) : "memory");
      asm volatile("cp.async.bulk.commit_group;" ::: "memory");
      asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");
    }
  }
  if (acc == 0x1234567ull) *sink = acc;
}

static cudaTextureObject_t g_tex;
static int g_sms = 132;
template <int V>
float run(State* st, Slot* dict, uint32_t mask, uint64_t rows, uint32_t G, unsigned long long* sink, int ctas_per_sm) {
  cudaEvent_t e0, e1; CK(cudaEventCreate(&e0)); CK(cudaEventCreate(&e1));
  float best = 1e30f;
  for (int rep = 0; rep < 4; rep++) {
    CK(cudaMemsetAsync(st, 0, (size_t)G * sizeof(State)));
    CK(cudaEventRecord(e0));
    k_bench<V><<<g_sms * ctas_per_sm, 512>>>(st, dict, mask, rows, G, sink, g_tex);
    CK(cudaEventRecord(e1)); CK(cudaEventSynchronize(e1)); CK(cudaGetLastError());
    float ms; CK(cudaEventElapsedTime(&ms, e0, e1)); if (rep && ms < best) best = ms;
  }
  return best;
}

int main(int argc, char** argv) {
  int lg = argc > 1 ? atoi(argv[1]) : 26; uint32_t G = argc > 2 ? (uint32_t)atoi(argv[2]) : 100000u;
  uint64_t rows = 1ull << lg;
  uint32_t gcap = 1; while (gcap < G) gcap <<= 1;
  const uint32_t cap = gcap * (gcap <= (1u << 20) ? 16u : gcap <= (8u << 20) ? 8u : 4u);     // dict_slots_per_group
  CK(cudaDeviceGetAttribute(&g_sms, cudaDevAttrMultiProcessorCount, 0));
  State* st; Slot* dict; unsigned long long* sink;
  CK(cudaMalloc(&st, (size_t)G * sizeof(State))); CK(cudaMalloc(&dict, (size_t)cap * sizeof(Slot))); CK(cudaMalloc(&sink, 8));
  CK(cudaMemset(dict, 0, (size_t)cap * sizeof(Slot)));
  {
    cudaResourceDesc rd{}; rd.resType = cudaResourceTypeLinear; rd.res.linear.devPtr = dict; rd.res.linear.desc = cudaCreateChannelDesc<uint4>();
    rd.res.linear.sizeInBytes = (size_t)cap * sizeof(Slot);
    cudaTextureDesc td{}; td.readMode = cudaReadModeElementType;
    CK(cudaCreateTextureObject(&g_tex, &rd, &td, nullptr));
  }
  cudaDeviceProp prop; CK(cudaGetDeviceProperties(&prop, 0));
  printf("%s, %d SMs, L2 %.0f MB | rows=2^%d groups=%u dict_slots=%u (%.1f MB) state=%.1f MB\n", prop.name, g_sms, prop.l2CacheSize / 1e6, lg, G,
         cap, cap * 32.0 / 1e6, G * 32.0 / 1e6);
  for (int cps = 1; cps <= 4; cps *= 2) {
    printf("--- %d CTA(s) of 512 threads per SM\n", cps);
    float ms[V_COUNT];
    ms[V_RED4] = run<V_RED4>(st, dict, cap - 1, rows, G, sink, cps);
    ms[V_RED2] = run<V_RED2>(st, dict, cap - 1, rows, G, sink, cps);
    ms[V_PAIR] = run<V_PAIR>(st, dict, cap - 1, rows, G, sink, cps);
    ms[V_PAIR_ADD] = run<V_PAIR_ADD>(st, dict, cap - 1, rows, G, sink, cps);
    ms[V_PROBE] = run<V_PROBE>(st, dict, cap - 1, rows, G, sink, cps);
    ms[V_PROBE_NC] = run<V_PROBE_NC>(st, dict, cap - 1, rows, G, sink, cps);
    ms[V_PROBE_RED4] = run<V_PROBE_RED4>(st, dict, cap - 1, rows, G, sink, cps);
    ms[V_PROBE_PAIR] = run<V_PROBE_PAIR>(st, dict, cap - 1, rows, G, sink, cps);
    ms[V_PROBE_HINT] = run<V_PROBE_HINT>(st, dict, cap - 1, rows, G, sink, cps);
    ms[V_PROBE_HINT_SCALAR] = run<V_PROBE_HINT_SCALAR>(st, dict, cap - 1, rows, G, sink, cps);
    ms[V_BULK] = run<V_BULK>(st, dict, cap - 1, rows, G, sink, cps);
    ms[V_QUAD_ADD] = run<V_QUAD_ADD>(st, dict, cap - 1, rows, G, sink, cps);
    ms[V_RED1] = run<V_RED1>(st, dict, cap - 1, rows, G, sink, cps);
    ms[V_PROBE_RED1] = run<V_PROBE_RED1>(st, dict, cap - 1, rows, G, sink, cps);
    ms[V_PROBE16] = run<V_PROBE16>(st, dict, cap - 1, rows, G, sink, cps);
    ms[V_TEX32] = run<V_TEX32>(st, dict, cap - 1, rows, G, sink, cps);
    ms[V_TEX16] = run<V_TEX16>(st, dict, cap - 1, rows, G, sink, cps);
    ms[V_TEX32_HINT] = run<V_TEX32_HINT>(st, dict, cap - 1, rows, G, sink, cps);
    ms[V_PROBE_HINT_XOR] = run<V_PROBE_HINT_XOR>(st, dict, cap - 1, rows, G, sink, cps);
    ms[V_XOR_ADD] = run<V_XOR_ADD>(st, dict, cap - 1, rows, G, sink, cps);
    ms[V_PROBE_PAIRED] = run<V_PROBE_PAIRED>(st, dict, cap - 1, rows, G, sink, cps);
    ms[V_PROBE_PAIRED_HINT_XOR] = run<V_PROBE_PAIRED_HINT_XOR>(st, dict, cap - 1, rows, G, sink, cps);
    for (int v = 0; v < V_COUNT; v++)
      printf("%-66s %8.3f ms  %7.1f G rows/s  %5.2f cyc/row/SM @1.9GHz\n", NAMES[v], ms[v], rows / ms[v] * 1e-6, ms[v] * 1e-3 * 1.9e9 * g_sms / rows);
  }
  return 0;
}
