// wdb_mlp.cu -- fused policy/value MLP forward on the Hopper tensor cores (wgmma).
//
// Replaces, for the rollout path, FullyConnected.forward of the reference
// (warp_drive/training/models/fully_connected.py:51-89): obs -> Linear+ReLU -> Linear+ReLU ->
// {head0 softmax, head1 softmax, value}.  The reference (and the torch fallback) runs it as
// 5 GEMMs + 7 elementwise kernels that round-trip the [rows, 256] activations through HBM;
// here one persistent kernel keeps them on chip:
//
//   * all weights (bf16, pre-packed by wdb_mlp_pack_weights into the wgmma canonical K-major
//     no-swizzle layout) are TMA-bulk-loaded into shared memory ONCE per CTA;
//   * every warpgroup owns 64 rows of a 128-row tile and runs the three layers on its own,
//     with no block-wide synchronisation inside the tile loop.  For the config-2 shape
//     (FastShape) every layer takes its A operand from registers (wgmma register-A form):
//     layer 1's fragments are loaded by each thread straight from the observations (fp32
//     rows or a bf16 obs tile).  Other shapes stage layer 1's operand in a per-warpgroup
//     shared-memory buffer.  Layers 2 and 3 always read registers: the fp32 accumulator fragment of
//     a hidden layer, after bias + ReLU + bf16 packing, IS the A fragment of the next layer,
//     so hidden activations never touch shared or global memory.  B is always read from
//     the shared-memory weights through a matrix descriptor;
//   * for the config-2 shape (FastShape) a hidden layer is computed in 64-column slices
//     (wgmma m64n64k16), pipelined: slice c + 1's MMAs run while slice c's epilogue packs it,
//     each packed slice of layer 2 feeds its four layer-3 k-steps (one m64n48k16 each) at
//     once, and the next tile's observations are loaded during layer 2.  Other shapes run
//     one 32-column slice (m64n32k16) at a time, holding both hidden layers' packed
//     activations;
//   * final epilogue = bias + two softmaxes + value: the logits go through the staging
//     buffer, two threads per row (head 0 | head 1 + value) compute the softmaxes, and the
//     warpgroup's 64 rows of each output are copied to global memory with coalesced stores.
//     The sampling forward (mlp_forward_sampled_kernel) gives this epilogue, and the
//     sampling of both heads, to a third warpgroup, so its two MMA warpgroups only run MMAs.
//
// Numerics: bf16 operands, fp32 accumulation (the reference is fp32; SURVEY.md section 8
// row a3 allows TF32/BF16 for the forward that feeds the sampler).  Pinned to a float64
// reference that emulates this quantisation (tests/mlp_reference.py, test_gpu_mlp_exact.py):
// on inputs whose fp32 dot products are exact, values bit-exact and probabilities within 1e-5
// relative; the weight blob and obs tiles byte-exact.  tests/test_gpu_mlp.py measures the gap
// to the float32 torch module (probabilities within 2e-2 abs).
#include <cuda_bf16.h>
#include <math_constants.h>

#include "wdb_common.cuh"

using namespace wdb;

namespace {

constexpr int kTileM = 128;            // rows of an obs tile (the wdb_mlp_pack_obs layout)
constexpr int kWgRows = 64;            // rows per warpgroup (wgmma M)
constexpr int kWarpgroups = kTileM / kWgRows;
constexpr int kThreads = 128 * kWarpgroups;
constexpr int kMaxK = 256;             // K1 and H are at most 256 (mlp_shape_ok)
constexpr int kMaxN3 = 64;             // A0 + A1 + 1 <= 64, padded to 16
constexpr int kMlpWeightsStable = 1;   // wdb_mlp_policy_forward_pair flags
__device__ __forceinline__ void griddep_wait() {
  asm volatile("griddepcontrol.wait;" ::: "memory");
}
__device__ __forceinline__ void griddep_launch_dependents() {
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
}

struct MlpHeader {            // start of the packed weight blob (device memory)
  int F, K1, H, A0, A1, N3;   // input features, padded K of layer 1, hidden width, heads, padded N3
  int off_w1, off_w2, off_w3, off_b, total_bytes, pad;
};
// Where the blob's parts start: header | W1 | W2 | W3 | biases.  A function of K1, H and N3
// alone, so a kernel compiled for one shape (FastShape) has them as constants.
struct MlpLayout {
  int off_w1, off_w2, off_w3, off_b, total_bytes;
};
__host__ __device__ constexpr MlpLayout mlp_layout(int K1, int H, int N3) {
  const int w1 = 128, w2 = w1 + H * K1 * 2, w3 = w2 + H * H * 2, b = w3 + N3 * H * 2;
  return {w1, w2, w3, b, (b + (2 * H + N3) * 4 + 15) / 16 * 16};
}

__device__ __forceinline__ uint32_t smem_addr(const void *p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

// wgmma shared-memory matrix descriptor, K-major, no swizzle ("interleaved" 8x16B core
// matrices): element (r, k) of a [rows, K] bf16 tile lives at
//   (r / 8) * SBO + (k / 8) * 128 + (r % 8) * 16 + (k % 8) * 2     [LBO = 128]
__device__ __forceinline__ uint64_t make_desc(uint32_t saddr, uint32_t sbo_bytes) {
  uint64_t d = 0;
  d |= (uint64_t)((saddr >> 4) & 0x3FFF);
  d |= (uint64_t)((128u >> 4) & 0x3FFF) << 16;
  d |= (uint64_t)((sbo_bytes >> 4) & 0x3FFF) << 32;
  return d;                   // layout_type = 0 (no swizzle), base_offset = 0
}

__device__ __forceinline__ void wgmma_fence() {
  asm volatile("wgmma.fence.sync.aligned;" ::: "memory");
}
__device__ __forceinline__ void wgmma_commit() {
  asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory");
}
// wait until at most N committed groups of this warp are still in flight
template <int N>
__device__ __forceinline__ void wgmma_wait() {
  asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory");
}

// The descriptor of make_desc, built inside the asm of a register-A wgmma from the 32-bit
// shared address ADDR and SBO / 16: computed next to its use, it is not hoisted out of the
// tile loop into (many) live 64-bit registers.
#define WGMMA_DESC_PTX(ADDR, SBO16)                                                    \
  "shr.b32 lo, " ADDR ", 4;\n\tand.b32 lo, lo, 0x3FFF;\n\tor.b32 lo, lo, 0x80000;\n\t" \
  "mov.b64 bd, {lo, " SBO16 "};\n\t"

// D[64 x 32] (+)= A[64 x 16] (shared memory, K-major) * B[16 x 32] (shared memory, K-major)
__device__ __forceinline__ void wgmma_n32_ss(float (&d)[16], uint64_t adesc, uint64_t bdesc,
                                             int accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %18, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n32k16.f32.bf16.bf16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, "
      "%16, %17, p, 1, 1, 0, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]),
        "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]),
        "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
      : "l"(adesc), "l"(bdesc), "r"(accumulate)
      : "memory");
}
// D[64 x 32] (+)= A[64 x 16] (registers, bf16) * B[16 x 32] (shared memory, K-major)
__device__ __forceinline__ void wgmma_n32(float (&d)[16], const uint32_t *a, uint32_t baddr,
                                          uint32_t bsbo, int accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t.reg .b32 lo;\n\t.reg .b64 bd;\n\tsetp.ne.b32 p, %22, 0;\n\t"
      WGMMA_DESC_PTX("%20", "%21")
      "wgmma.mma_async.sync.aligned.m64n32k16.f32.bf16.bf16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, "
      "{%16, %17, %18, %19}, bd, p, 1, 1, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]),
        "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]),
        "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(baddr), "r"(bsbo >> 4), "r"(accumulate)
      : "memory");
}
// D[64 x 64] (+)= A[64 x 16] (registers, bf16) * B[16 x 64] (shared memory, K-major)
__device__ __forceinline__ void wgmma_n64(float (&d)[32], const uint32_t *a, uint32_t baddr,
                                          uint32_t bsbo, int accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t.reg .b32 lo;\n\t.reg .b64 bd;\n\tsetp.ne.b32 p, %38, 0;\n\t"
      WGMMA_DESC_PTX("%36", "%37")
      "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
      "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, "
      "{%32, %33, %34, %35}, bd, p, 1, 1, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]),
        "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]),
        "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]),
        "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]),
        "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]),
        "+f"(d[31])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(baddr), "r"(bsbo >> 4), "r"(accumulate)
      : "memory");
}
// D[64 x 48] (+)= A[64 x 16] (registers, bf16) * B[16 x 48] (shared memory, K-major)
__device__ __forceinline__ void wgmma_n48(float (&d)[24], const uint32_t *a, uint32_t baddr,
                                          uint32_t bsbo, int accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t.reg .b32 lo;\n\t.reg .b64 bd;\n\tsetp.ne.b32 p, %30, 0;\n\t"
      WGMMA_DESC_PTX("%28", "%29")
      "wgmma.mma_async.sync.aligned.m64n48k16.f32.bf16.bf16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
      "%16, %17, %18, %19, %20, %21, %22, %23}, "
      "{%24, %25, %26, %27}, bd, p, 1, 1, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]),
        "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]),
        "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]),
        "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(baddr), "r"(bsbo >> 4), "r"(accumulate)
      : "memory");
}
// D[64 x 16] (+)= A[64 x 16] * B[16 x 16]
__device__ __forceinline__ void wgmma_n16(float (&d)[8], const uint32_t *a, uint32_t baddr,
                                          uint32_t bsbo, int accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t.reg .b32 lo;\n\t.reg .b64 bd;\n\tsetp.ne.b32 p, %14, 0;\n\t"
      WGMMA_DESC_PTX("%12", "%13")
      "wgmma.mma_async.sync.aligned.m64n16k16.f32.bf16.bf16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7}, {%8, %9, %10, %11}, bd, p, 1, 1, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]),
        "+f"(d[7])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(baddr), "r"(bsbo >> 4), "r"(accumulate)
      : "memory");
}

__device__ __forceinline__ void mbar_init(uint32_t mbar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(mbar), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t mbar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(mbar), "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void mbar_wait(uint32_t mbar, uint32_t parity) {
  uint32_t ok;
  do {
    asm volatile(
        "{ .reg .pred p; mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2; "
        "selp.u32 %0, 1, 0, p; }"
        : "=r"(ok) : "r"(mbar), "r"(parity) : "memory");
  } while (!ok);
}
__device__ __forceinline__ void tma_load(uint32_t dst, const void *src, uint32_t bytes,
                                         uint32_t mbar) {
  asm volatile(
      "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
      ::"r"(dst), "l"(src), "r"(bytes), "r"(mbar) : "memory");
}

__device__ __forceinline__ uint32_t pack_bf16(float lo, float hi) {
  const __nv_bfloat162 h = __floats2bfloat162_rn(lo, hi);
  return *reinterpret_cast<const uint32_t *>(&h);
}

// (lo + b_lo, hi + b_hi) -> ReLU -> packed bf16x2
__device__ __forceinline__ uint32_t bias_relu_pack(float lo, float hi, float b_lo, float b_hi) {
  uint32_t out;
  asm("cvt.rn.relu.bf16x2.f32 %0, %1, %2;" : "=r"(out) : "f"(hi + b_hi), "f"(lo + b_lo));
  return out;
}

// named barrier of one warpgroup (ids 1, 2; 0 is __syncthreads)
__device__ __forceinline__ void wg_sync(int wg) {
  if (wg) asm volatile("bar.sync 2, 128;" ::: "memory");
  else asm volatile("bar.sync 1, 128;" ::: "memory");
}

// dst[0 .. n) = src[0 .. n) by the 128 threads of a warpgroup (lt = thread in it); src is
// 16-byte aligned, so when dst is too the bulk moves as float4
__device__ __forceinline__ void copy_out(float *__restrict__ dst, const float *src, int n,
                                         int lt) {
  int done = 0;
  if ((reinterpret_cast<uintptr_t>(dst) & 15) == 0) {
    done = n & ~3;
    for (int i = lt; i < n / 4; i += 128)
      reinterpret_cast<float4 *>(dst)[i] = reinterpret_cast<const float4 *>(src)[i];
  }
  for (int i = done + lt; i < n; i += 128) dst[i] = src[i];
}

// A hidden layer of a warpgroup is computed in kSliceN-column slices (wgmma m64n64k16, one
// commit group per slice) with two accumulator sets: slice c + 1's MMAs are issued before
// the epilogue of slice c (`epi`) runs, so the tensor cores always have a slice in flight.
// issue(c, d) issues slice c into d; its first MMA
// runs with scale-d = 0, so the accumulators need no zeroing (a zeroing store between the
// fence and the MMAs would serialise the pipeline).  epi(c, d) may itself commit MMA groups:
// the wait before slice c's epilogue leaves only slice c + 1 in flight.
// Accumulator fragment of m64nNk16: lane (g = lane / 4, t = lane % 4) of warp w holds rows
// 16 w + g (+ 8), columns 8 j + 2 t (+ 1); the k-step kk of the next layer's A fragment is
// columns 16 kk .. 16 kk + 15 of the same rows in the same lanes, so the repacking is
// register-to-register.
constexpr int kSliceN = 64;
template <class Issue, class Epi>
__device__ __forceinline__ void slice_pipeline(int n_slices, Issue issue, Epi epi) {
  float d[2][kSliceN / 2];
  wgmma_fence();
  issue(0, d[0]);
  wgmma_commit();
#pragma unroll
  for (int c = 0; c < kMaxK / kSliceN; c++) {
    if (c < n_slices) {
      if (c + 1 < n_slices) {
        wgmma_fence();                 // (slice c - 1's epilogue read this accumulator set)
        issue(c + 1, d[(c + 1) & 1]);
        wgmma_commit();
        wgmma_wait<1>();
      } else {
        wgmma_wait<0>();
      }
      epi(c, d[c & 1]);
    }
  }
}

// slice c of a hidden layer's accumulators + bias -> ReLU -> packed bf16 A fragments
// out[0 .. kSliceN / 4) (the next layer's k-steps kSliceN / 16 * c .. + kSliceN / 16 - 1)
__device__ __forceinline__ void bias_relu_slice(const float (&d)[kSliceN / 2], const float *bias,
                                                int c, uint32_t *out) {
  const int t = threadIdx.x & 3;
#pragma unroll
  for (int j = 0; j < kSliceN / 8; j++) {
    const float2 b = *reinterpret_cast<const float2 *>(bias + kSliceN * c + 8 * j + 2 * t);
    out[2 * j] = bias_relu_pack(d[4 * j], d[4 * j + 1], b.x, b.y);
    out[2 * j + 1] = bias_relu_pack(d[4 * j + 2], d[4 * j + 3], b.x, b.y);
  }
}

// One hidden layer of a warpgroup, one slice at a time (the schedule of runtime shapes):
// out (packed bf16 A fragments of the next layer, 4 per
// 16 columns) = ReLU(A * W^T + bias), W = [N, K] in the canonical K-major layout at shared
// address w.  A (K / 16 k-steps) is `in` (register fragments) or, with SS, the canonical
// tile at the shared address a_smem (row-group stride a_sbo).  Accumulator fragment
// of m64nNk16: lane (g = lane / 4, t = lane % 4) of warp w holds rows 16 w + g (+ 8),
// columns 8 j + 2 t (+ 1); the k-step kk of the next layer's A fragment is columns
// 16 kk .. 16 kk + 15 of the same rows in the same lanes, so the repacking is
// register-to-register (see bias_relu_slice).  Scale-d = 0 on the first MMA of a slice,
// as in slice_pipeline.
template <bool SS>
__device__ __forceinline__ void hidden_layer(const uint32_t (&in)[kMaxK / 4], uint32_t a_smem,
                                             uint32_t a_sbo, int K, uint32_t w, uint32_t sbo,
                                             int N, const float *bias,
                                             uint32_t (&out)[kMaxK / 4]) {
  const int t = threadIdx.x & 3;
#pragma unroll
  for (int c = 0; c < kMaxK / 32; c++) {
    if (c < N / 32) {
      float d[16];
      wgmma_fence();
      if (SS) {
        for (int kk = 0; kk < K / 16; kk++)
          wgmma_n32_ss(d, make_desc(a_smem + kk * 256, a_sbo),
                       make_desc(w + 4 * c * sbo + kk * 256, sbo), kk);
      } else {
#pragma unroll
        for (int kk = 0; kk < kMaxK / 16; kk++)
          if (kk < K / 16) wgmma_n32(d, &in[4 * kk], w + 4 * c * sbo + kk * 256, sbo, kk);
      }
      wgmma_commit();
      wgmma_wait<0>();
#pragma unroll
      for (int j = 0; j < 4; j++) {
        const float2 b = *reinterpret_cast<const float2 *>(bias + 32 * c + 8 * j + 2 * t);
        out[8 * c + 2 * j] = bias_relu_pack(d[4 * j], d[4 * j + 1], b.x, b.y);
        out[8 * c + 2 * j + 1] = bias_relu_pack(d[4 * j + 2], d[4 * j + 3], b.x, b.y);
      }
    }
  }
}

// ---- layer-1 A operand of the FastShape schedule, in register-A form: each thread loads the
// elements of its own A fragments straight from the observations, so the operand never
// passes through shared memory.  Fragment 4 kk + q of k-step kk (the layout of
// bias_relu_slice's output) holds row 16 w + g (q = 0, 2) or 16 w + g + 8 (q = 1, 3),
// columns 16 kk + 2 t (+ 1) (q = 0, 1) or 16 kk + 8 + 2 t (+ 1) (q = 2, 3), as bf16x2.
// A thread's loads for the NEXT tile are issued during the current tile's layer 2 and packed
// a slice later (obs_frag_pack), in two halves (part 0: fragments [0, K1 / 8), part 1 the
// rest), so at most half of the operand is live unpacked.
template <bool TILES, int K1> struct ObsFrag;
template <int K1> struct ObsFrag<false, K1> { float v[K1 / 8][2]; };   // fp32 obs [rows, F]
template <int K1> struct ObsFrag<true, K1> { uint32_t v[K1 / 8]; };    // bf16 obs tiles

// rows beyond `rows` and columns >= F read as 0 (the zero padding of the staged operand)
template <int K1>
__device__ __forceinline__ void obs_frag_load(ObsFrag<false, K1> &f, int part,
                                              const void *input, long long rows, int F,
                                              long long row0) {
  const int wr = (threadIdx.x >> 5) & 3, g = (threadIdx.x >> 2) & 7, t = threadIdx.x & 3;
#pragma unroll
  for (int j = 0; j < K1 / 8; j++) {
    const int i = part * (K1 / 8) + j;
    const long long row = row0 + 16 * wr + g + 8 * (i & 1);
    const int col = 16 * (i >> 2) + 8 * ((i >> 1) & 1) + 2 * t;
    const float *src = reinterpret_cast<const float *>(input) + row * F + col;
    f.v[j][0] = (row < rows && col < F) ? __ldg(src) : 0.0f;
    f.v[j][1] = (row < rows && col + 1 < F) ? __ldg(src + 1) : 0.0f;
  }
}
// the warpgroup's 64 rows are one contiguous block of a tile in the canonical K-major layout
// ((r, k) at (r / 8) * K1 * 16 + (k / 8) * 128 + (r % 8) * 16 + (k % 8) * 2; rows past the
// end are the zero padding of the tile buffer), so a fragment is one aligned 4-byte word
template <int K1>
__device__ __forceinline__ void obs_frag_load(ObsFrag<true, K1> &f, int part,
                                              const void *input, long long, int,
                                              long long row0) {
  const int wr = (threadIdx.x >> 5) & 3, g = (threadIdx.x >> 2) & 7, t = threadIdx.x & 3;
  const unsigned char *src =
      reinterpret_cast<const unsigned char *>(input) + row0 * (K1 * 2) + g * 16 + t * 4;
#pragma unroll
  for (int j = 0; j < K1 / 8; j++) {
    const int i = part * (K1 / 8) + j;
    const int grp = 2 * wr + (i & 1), chunk = 2 * (i >> 2) + ((i >> 1) & 1);
    f.v[j] = __ldg(reinterpret_cast<const uint32_t *>(src + grp * (K1 * 16) + chunk * 128));
  }
}
template <int K1>
__device__ __forceinline__ void obs_frag_pack(const ObsFrag<false, K1> &f, int part,
                                              uint32_t (&a)[K1 / 4]) {
#pragma unroll
  for (int j = 0; j < K1 / 8; j++) a[part * (K1 / 8) + j] = pack_bf16(f.v[j][0], f.v[j][1]);
}
template <int K1>
__device__ __forceinline__ void obs_frag_pack(const ObsFrag<true, K1> &f, int part,
                                              uint32_t (&a)[K1 / 4]) {
#pragma unroll
  for (int j = 0; j < K1 / 8; j++) a[part * (K1 / 8) + j] = f.v[j];
}

// Profiling aid (-DWDB_PHASE_CLOCKS): thread 0 of CTA 0 of one forward launch at a time
// records clock64 at the phase boundaries, read back by wdb_debug_mlp_clocks.  [0] = rows of
// the recorded launch, [1] kernel start, [2] weights landed, then per tile k < 18 of the CTA,
// [3 + 5 k + p]: p = 0 tile start, 1 layer 1 done, 2 layers 2 + 3 done, 3 softmax done,
// 4 outputs stored.
#ifdef WDB_PHASE_CLOCKS
constexpr int kMlpClockSlots = 96;
__device__ long long g_mlp_clocks[kMlpClockSlots];
__device__ int g_mlp_clocks_busy;
#define MLP_MARK(i)                                                                  \
  if (rec_clocks && (i) < kMlpClockSlots) g_mlp_clocks[(i)] = clock64();
#else
#define MLP_MARK(i)
#endif

// TILES = false: `input` is the fp32 obs [rows, F]; TILES = true: `input` is the bf16 copy of
// the obs already in A-operand layout (128-row tiles of the canonical K-major layout, K
// padded with zeros -- written by wdb_mlp_pack_obs or by the env-step kernel's epilogue).
// `bid` / `gdim`: this CTA's index and the CTA count of ITS policy (the pair kernel runs two
// policies side by side in one grid).  flags & kMlpWeightsStable: the weight blob was not
// written by the grid this launch programmatically depends on, so its TMA load may start
// before griddepcontrol.wait (see the PDL note at launch_forward_pair).
// Shape: MlpShape<0, 0, 0> reads K1, H and N3 from the blob's header; a non-zero shape is
// the header's, fixed at compile time (FastShape).
// MASK: `mask` [rows, A0 + A1] marks the valid actions (wdb_mlp_policy_forward_masked); the
// unmasked instantiations compile without any of its code.
template <int K1_, int H_, int N3_> struct MlpShape {
  static constexpr int K1 = K1_, H = H_, N3 = N3_;
};
using AnyShape = MlpShape<0, 0, 0>;
// The config-2 policies (F = 71 -> K1 = 80, H = 256, 21 + 21 + 1 -> N3 = 48).  With every
// MMA loop bound a constant, ptxas can follow the wgmma groups of the overlapped schedule
// (slice_pipeline, the next tile's observations prefetched during layer 2): it keeps
// slice c + 1's MMAs in flight across slice c's epilogue and injects no warpgroup.arrive.
// With runtime bounds it would serialise those wgmmas (C7514) and the extra live registers
// would spill, so every other shape runs one slice at a time and loads its observations
// at the top of the tile.
using FastShape = MlpShape<80, 256, 48>;

// ---- the FastShape schedule of one warpgroup's tile, in two parts (the caller marks the
// phase clock between them).  Layer 1 (A = a1, in registers) -> h: packed bf16 A fragments
// of layer 2.
__device__ __forceinline__ void fast_layer1(const uint32_t (&a1)[FastShape::K1 / 4],
                                            uint32_t s_w1, uint32_t sbo_a, const float *s_b1,
                                            uint32_t (&h)[kMaxK / 4]) {
  slice_pipeline(
      FastShape::H / kSliceN,
      [&](int c, float(&d)[kSliceN / 2]) {
#pragma unroll
        for (int kk = 0; kk < FastShape::K1 / 16; kk++)
          wgmma_n64(d, &a1[4 * kk], s_w1 + kSliceN / 8 * c * sbo_a + kk * 256, sbo_a, kk);
      },
      [&](int c, const float(&d)[kSliceN / 2]) {
        bias_relu_slice(d, s_b1, c, &h[kSliceN / 4 * c]);
      });
}

// Layer 2 (A = h) streamed into layer 3 ([head0 | head1 | value | pad], one m64n48k16 per
// k-step, accumulated in o48): as soon as a 64-column slice of layer 2 is packed, the four
// layer-3 k-steps it feeds are issued, so layer 2's output is never held whole.  Every
// layer-3 output still accumulates its k-steps 0, 1, ..., H / 16 - 1 in order, the first
// with scale-d = 0.  The n48 accumulator fragment holds columns 8 j + 2 t (+ 1) at [4 j ..].
// When have_next, the observations of the warpgroup's next tile (first row next_row0) load
// meanwhile, half after slice 0 and half after slice 1, each packed into a1 (which layer 1
// no longer reads) one slice after its loads were issued.  Returns with layer 3's MMAs
// still in flight (the caller's wgmma_wait<0> completes o48).
template <bool TILES>
__device__ __forceinline__ void fast_layers23(const uint32_t (&h)[kMaxK / 4], uint32_t s_w2,
                                              uint32_t s_w3, uint32_t sbo_h, const float *s_b2,
                                              float (&o48)[48 / 2],
                                              ObsFrag<TILES, FastShape::K1> &next,
                                              uint32_t (&a1)[FastShape::K1 / 4], bool have_next,
                                              const void *input, long long rows, int F,
                                              long long next_row0) {
  slice_pipeline(
      FastShape::H / kSliceN,
      [&](int c, float(&d)[kSliceN / 2]) {
#pragma unroll
        for (int kk = 0; kk < FastShape::H / 16; kk++)
          wgmma_n64(d, &h[4 * kk], s_w2 + kSliceN / 8 * c * sbo_h + kk * 256, sbo_h, kk);
      },
      [&](int c, const float(&d)[kSliceN / 2]) {
        uint32_t a[kSliceN / 4];
        bias_relu_slice(d, s_b2, c, a);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < kSliceN / 16; k++)
          wgmma_n48(o48, &a[4 * k], s_w3 + (kSliceN / 16 * c + k) * 256, sbo_h,
                    kSliceN / 16 * c + k);
        wgmma_commit();
        if (have_next && (c == 1 || c == 2)) obs_frag_pack(next, c - 1, a1);
        if (have_next && (c == 0 || c == 1)) obs_frag_load(next, c, input, rows, F, next_row0);
      });
}

// ---- output epilogue of a warpgroup's 64 rows.  The logits are staged [64 rows x N3] with
// column col of row r at col ^ (r & 14): the softmax reads one column of 32 consecutive rows
// per warp, which with N3 = 48 would otherwise fall into two shared-memory banks (16-way
// conflicts; 2-way with it).  The swizzle stays inside the column's 16-column group (N3 is a
// multiple of 16) and keeps the pairs (col, col + 1) of even col together, so they are still
// float2 stores.
__device__ __forceinline__ int logit_at(int r, int col, int N3) {
  return r * N3 + (col ^ (r & 14));
}

// layer 3's accumulators + bias -> staging: o[c][4 j + 0/1] is row lr = 16 wr + g,
// o[c][4 j + 2/3] row lr + 8, columns 16 c + 8 j + 2 t (+1)
__device__ __forceinline__ void stage_logits(const float (&o)[kMaxN3 / 16][8], const float *s_b3,
                                             int N3, int lr, int t, float *s_o) {
#pragma unroll
  for (int c = 0; c < kMaxN3 / 16; c++) {
    if (c < N3 / 16) {
#pragma unroll
      for (int j = 0; j < 2; j++) {
        const int col = 16 * c + 8 * j + 2 * t;
        const float2 b = *reinterpret_cast<const float2 *>(s_b3 + col);
        *reinterpret_cast<float2 *>(s_o + logit_at(lr, col, N3)) =
            make_float2(o[c][4 * j] + b.x, o[c][4 * j + 1] + b.y);
        *reinterpret_cast<float2 *>(s_o + logit_at(lr + 8, col, N3)) =
            make_float2(o[c][4 * j + 2] + b.x, o[c][4 * j + 3] + b.y);
      }
    }
  }
}

// Softmax of the cnt staged logits of `row` from column cbase: lg[i] = 2^(l_i log2(e) - max)
// (0 for i >= cnt), returns 1 / sum; `value` = the logit just past the head (the value
// column, for head 1).  Logits pre-scaled by log2(e), branch-free over 32 statically indexed
// registers, 4-way max and sum.
__device__ __forceinline__ float softmax_row(const float *s_o, int N3, int row, int cbase,
                                             int cnt, float (&lg)[32], float &value) {
  constexpr float kLog2e = 1.4426950408889634f;
  float mx[4] = {-CUDART_INF_F, -CUDART_INF_F, -CUDART_INF_F, -CUDART_INF_F};
  value = 0.0f;
#pragma unroll
  for (int i = 0; i < 32; i++) {
    const float x = s_o[logit_at(row, min(cbase + i, N3 - 1), N3)];
    lg[i] = i < cnt ? x * kLog2e : -CUDART_INF_F;
    mx[i & 3] = fmaxf(mx[i & 3], lg[i]);
    value = (i == cnt) ? x : value;
  }
  const float m = fmaxf(fmaxf(mx[0], mx[1]), fmaxf(mx[2], mx[3]));
  float zz[4] = {0.0f, 0.0f, 0.0f, 0.0f};
#pragma unroll
  for (int i = 0; i < 32; i++) {
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(lg[i]) : "f"(lg[i] - m));   // 2^-inf = 0
    zz[i & 3] += lg[i];
  }
  return 1.0f / ((zz[0] + zz[1]) + (zz[2] + zz[3]));
}

// staged [probs0 64 x A0 | probs1 64 x A1 | values 64] of the 64 rows from rb -> global
__device__ __forceinline__ void copy_outputs(const float *s_o, long long rb, long long rows,
                                             int A0, int A1, float *__restrict__ probs0,
                                             float *__restrict__ probs1,
                                             float *__restrict__ values, int lt) {
  const float *s_p0 = s_o, *s_p1 = s_o + kWgRows * A0, *s_v = s_p1 + kWgRows * A1;
  const int valid = (int)min((long long)kWgRows, rows - rb);
  copy_out(probs0 + rb * A0, s_p0, valid * A0, lt);
  copy_out(probs1 + rb * A1, s_p1, valid * A1, lt);
  if (values && lt < valid) values[rb + lt] = s_v[lt];
}

template <bool TILES, class Shape, bool MASK = false>
__device__ __forceinline__ void
mlp_forward_body(const unsigned char *__restrict__ blob, const void *__restrict__ input,
                 long long rows, float *__restrict__ probs0, float *__restrict__ probs1,
                 float *__restrict__ values, const unsigned bid, const unsigned gdim,
                 const int flags, const float *__restrict__ mask = nullptr) {
  extern __shared__ __align__(128) unsigned char smem[];
  const MlpHeader hd = *reinterpret_cast<const MlpHeader *>(blob);
  const int F = hd.F, A0 = hd.A0, A1 = hd.A1;
  const int K1 = Shape::K1 ? Shape::K1 : hd.K1, H = Shape::H ? Shape::H : hd.H,
            N3 = Shape::N3 ? Shape::N3 : hd.N3;
  constexpr bool kOverlap = Shape::H != 0;
  // FastShape: constant offsets, so the wgmma descriptors fold to constants (computed from
  // the header they take registers, and the fp32-observation kernel spills)
  const MlpLayout lay = kOverlap ? mlp_layout(Shape::K1, Shape::H, Shape::N3)
                                 : MlpLayout{hd.off_w1, hd.off_w2, hd.off_w3, hd.off_b,
                                             hd.total_bytes};
  const int w_bytes = lay.total_bytes - lay.off_w1;      // W1 | W2 | W3 | biases, contiguous
  unsigned char *s_w = smem;                             // packed weights + biases
  const uint32_t s_w1 = smem_addr(s_w);
  const uint32_t s_w2 = s_w1 + (lay.off_w2 - lay.off_w1);
  const uint32_t s_w3 = s_w1 + (lay.off_w3 - lay.off_w1);
  const float *s_b1 = reinterpret_cast<const float *>(s_w + (lay.off_b - lay.off_w1));
  const float *s_b2 = s_b1 + H;
  const float *s_b3 = s_b2 + H;
  const int tid = threadIdx.x, lane = tid & 31;
  const int wg = tid >> 7, wr = (tid >> 5) & 3;          // warpgroup, warp within it
  const int g = lane >> 2, t = lane & 3;
  const int a_bytes = kWgRows * K1 * 2;                  // layer-1 A operand of one warpgroup
  const int stage_bytes = max(a_bytes, kWgRows * N3 * 4);   // ... or its logits / outputs
  unsigned char *s_a = s_w + ((w_bytes + 127) & ~127) + wg * stage_bytes;
  float *s_o = reinterpret_cast<float *>(s_a);
  unsigned long long *s_bar = reinterpret_cast<unsigned long long *>(
      s_w + ((w_bytes + 127) & ~127) + kWarpgroups * stage_bytes);
  const uint32_t bar_w = smem_addr(s_bar);               // weights landed
#ifdef WDB_PHASE_CLOCKS
  const bool rec_clocks = bid == 0 && tid == 0 && atomicCAS(&g_mlp_clocks_busy, 0, 1) == 0;
  if (rec_clocks) {
    for (int i = 0; i < kMlpClockSlots; i++) g_mlp_clocks[i] = 0;
    g_mlp_clocks[0] = rows;
  }
  int clock_tile = 0;
#endif
  MLP_MARK(1);
  if (tid == 0) {
    mbar_init(bar_w, 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  // Programmatic dependent launch: everything above overlapped the tail of the previous grid
  // in the stream.  Nothing that grid wrote is read before griddepcontrol.wait; our own
  // dependents are released only AFTER our wait, so "previous grid complete" is transitive.
  if (!(flags & kMlpWeightsStable)) griddep_wait();
  if (tid == 0) {                                         // weights: TMA bulk copies
    mbar_expect_tx(bar_w, (uint32_t)w_bytes);
    uint32_t off = 0;
    while (off < (uint32_t)w_bytes) {
      const uint32_t n = min((uint32_t)w_bytes - off, 65536u);
      tma_load(s_w1 + off, blob + lay.off_w1 + off, n, bar_w);
      off += n;
    }
  }
  if (flags & kMlpWeightsStable) griddep_wait();
  griddep_launch_dependents();

  const int lt = tid & 127;
  const long long n_tiles = (rows + kTileM - 1) / kTileM;
  // kOverlap: layer 1's A fragments of the warpgroup's current tile (a1), and the loads of its
  // next tile (next), issued during layer 2
  constexpr int kFragK1 = kOverlap ? Shape::K1 : 16;
  ObsFrag<TILES, kFragK1> next;
  uint32_t a1[kFragK1 / 4];
  const bool have_first = bid < n_tiles && bid * kTileM + wg * kWgRows < rows;
  if (kOverlap && have_first)                              // (overlaps the weight load)
    obs_frag_load(next, 0, input, rows, F, bid * kTileM + wg * kWgRows);
  mbar_wait(bar_w, 0);
  MLP_MARK(2);
  if (kOverlap && have_first) {
    obs_frag_pack(next, 0, a1);
    obs_frag_load(next, 1, input, rows, F, bid * kTileM + wg * kWgRows);
    obs_frag_pack(next, 1, a1);
  }

  const uint32_t sbo_a = (uint32_t)(K1 / 8) * 128u;       // W1: K1/8 core matrices per row group
  const uint32_t sbo_h = (uint32_t)(H / 8) * 128u;        // W2 / W3: H/8 core matrices per row group
  for (long long tile = bid; tile < n_tiles; tile += gdim) {
    const long long row0 = tile * kTileM + wg * kWgRows;  // first row of the warpgroup
    if (row0 >= rows) continue;                           // (warpgroup-uniform; so are all later tiles)
#ifdef WDB_PHASE_CLOCKS
    const int mark0 = 3 + 5 * (clock_tile < 18 ? clock_tile : kMlpClockSlots);
    clock_tile++;
#endif
    MLP_MARK(mark0);

    float o[kMaxN3 / 16][8];   // layer-3 logits
    if constexpr (kOverlap) {
      static_assert(Shape::K1 == FastShape::K1 && Shape::H == FastShape::H &&
                    Shape::N3 == FastShape::N3, "the overlapped schedule is FastShape's");
      uint32_t h[kMaxK / 4];
      fast_layer1(a1, s_w1, sbo_a, s_b1, h);
      MLP_MARK(mark0 + 1);
      // layer 3's n48 fragment (columns 8 j + 2 t (+ 1) at [4 j ..]) is o[n][4 j' ..]
      // (columns 16 n + 8 j' + 2 t) laid out flat
      float(&o48)[48 / 2] = *reinterpret_cast<float(*)[48 / 2]>(&o[0][0]);
      fast_layers23<TILES>(h, s_w2, s_w3, sbo_h, s_b2, o48, next, a1,
                           row0 + (long long)gdim * kTileM < rows, input, rows, F,
                           row0 + (long long)gdim * kTileM);
      wgmma_wait<0>();
    } else {
      // ---- layer 1 A operand -> this warpgroup's staging buffer (canonical K-major layout:
      // (r, k) at (r / 8) * K1 * 16 + (k / 8) * 128 + (r % 8) * 16 + (k % 8) * 2).  The
      // previous tile's layer-1 MMAs have completed (wait_group 0) in every warp.
      wg_sync(wg);
      if (TILES) {
        // the warpgroup's 64 rows are one contiguous block of the tile
        const uint4 *src = reinterpret_cast<const uint4 *>(
            reinterpret_cast<const unsigned char *>(input) + row0 * (K1 * 2));
        for (int i = lt; i < a_bytes / 16; i += 128)
          reinterpret_cast<uint4 *>(s_a)[i] = __ldg(src + i);
      } else {
        // task = one 16-byte chunk (8 consecutive k) of one row; consecutive lanes take the
        // 8 rows of a core matrix, so each shared store of a warp is bank-conflict free
        const int nchunk = K1 / 8;
        for (int i = lt; i < kWgRows * nchunk; i += 128) {
          const int grp = i / (8 * nchunk), in = i - grp * 8 * nchunk;
          const int c = in >> 3, r = 8 * grp + (in & 7);
          const long long row = row0 + r;
          const float *src = reinterpret_cast<const float *>(input) + row * F + 8 * c;
          float v[8];
#pragma unroll
          for (int k = 0; k < 8; k++) v[k] = (row < rows && 8 * c + k < F) ? __ldg(src + k) : 0.0f;
          uint4 o4;
          o4.x = pack_bf16(v[0], v[1]); o4.y = pack_bf16(v[2], v[3]);
          o4.z = pack_bf16(v[4], v[5]); o4.w = pack_bf16(v[6], v[7]);
          *reinterpret_cast<uint4 *>(s_a + grp * (K1 * 16) + c * 128 + (r & 7) * 16) = o4;
        }
      }
      asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // visible to wgmma
      wg_sync(wg);

      uint32_t a[kMaxK / 4], h[kMaxK / 4];
      hidden_layer<true>(a, smem_addr(s_a), sbo_a, K1, s_w1, sbo_a, H, s_b1, h);   // layer 1
      hidden_layer<false>(h, 0, 0, H, s_w2, sbo_h, H, s_b2, a);                     // layer 2

      // ---- layer 3: [head0 | head1 | value | pad] in 16-column slices
      wgmma_fence();
#pragma unroll
      for (int c = 0; c < kMaxN3 / 16; c++) {
        if (c < N3 / 16) {
#pragma unroll
          for (int kk = 0; kk < kMaxK / 16; kk++)
            if (kk < H / 16)
              wgmma_n16(o[c], &a[4 * kk], s_w3 + 2 * c * sbo_h + kk * 256, sbo_h, kk);
        }
      }
      wgmma_commit();
      wgmma_wait<0>();
    }
    MLP_MARK(mark0 + 2);

    // ---- output epilogue: logits (+ bias) -> staging, softmax, probabilities -> staging ->
    // global.  (The previous tile's output copy and, for other shapes, the layer-1 MMAs that
    // read the staging buffer have completed in every warp.)
    wg_sync(wg);
    stage_logits(o, s_b3, N3, wr * 16 + g, t, s_o);
    wg_sync(wg);
    if constexpr (MASK) {
      // apply_logit_mask in fp32 before the max: logit + (1 - m) * -1e20.  The warpgroup's
      // mask rows are one contiguous block, read coalesced like copy_out writes.
      const int am = A0 + A1;
      const long long mb = tile * kTileM + wg * kWgRows;
      const int n = (int)min((long long)kWgRows, rows - mb) * am;
      const float *src = mask + mb * am;
      for (int i = lt; i < n; i += 128) {
        const int r = i / am, col = i - r * am;
        float &x = s_o[logit_at(r, col, N3)];
        x = __fadd_rn(x, __fmul_rn(1.0f - __ldg(src + i), -1.0e20f));
      }
      wg_sync(wg);
    }
    // thread lt: row lt % 64; lt < 64 head 0, else head 1 + the value
    const int row = lt & 63, part = lt >> 6;
    const int cbase = part ? A0 : 0, cnt = part ? A1 : A0;
    float lg[32], value;
    const float inv = softmax_row(s_o, N3, row, cbase, cnt, lg, value);
    MLP_MARK(mark0 + 3);
    wg_sync(wg);
    // staging = [probs0 64 x A0 | probs1 64 x A1 | values 64]: the warpgroup's rows of each
    // output are contiguous in global memory
    float *s_p0 = s_o, *s_p1 = s_o + kWgRows * A0, *s_v = s_p1 + kWgRows * A1;
    float *dst = (part ? s_p1 : s_p0) + row * cnt;
#pragma unroll
    for (int i = 0; i < 32; i++)
      if (i < cnt) dst[i] = lg[i] * inv;
    if (part) s_v[row] = value;
    wg_sync(wg);
    copy_outputs(s_o, tile * kTileM + wg * kWgRows, rows, A0, A1, probs0, probs1, values, lt);
    MLP_MARK(mark0 + 4);
  }
#ifdef WDB_PHASE_CLOCKS
  if (rec_clocks) {
    __threadfence();
    atomicExch(&g_mlp_clocks_busy, 0);
  }
#endif
}

template <bool TILES, class Shape>
__global__ void __launch_bounds__(kThreads, 1)
mlp_forward_kernel(const unsigned char *__restrict__ blob, const void *__restrict__ input,
                   long long rows, float *__restrict__ probs0, float *__restrict__ probs1,
                   float *__restrict__ values, int flags) {
  mlp_forward_body<TILES, Shape>(blob, input, rows, probs0, probs1, values, blockIdx.x, gridDim.x, flags);
}

// ---- The sampling forward (FastShape only, wdb_mlp_policy_forward_sampled): besides the
// probabilities and values it draws both heads' actions of every row, as the fused
// TagContinuous step would from the stored probabilities.  Row r of the launch is row
// row0 + r = env * Np + slot of the policy, agent gi = env * N + agent[slot].
struct MlpSampling {
  int *actions;               // [rows, 2]
  void *rng;                  // RNG state of E * N streams (NULL with uniforms)
  const float *uniforms;      // [E * N * 2] or NULL
  const int *agent;           // [Np]
  int N, Np;
  long long row0;             // the launch's first row among the policy's rows
};

// Three warpgroups with fixed roles.  Warpgroups 0 and 1 each own 64 rows of every 128-row
// tile: they run the FastShape schedule of mlp_forward_body on them, then the softmax, and
// stage the probabilities and values in their staging buffer.  Warpgroup 2 draws both heads'
// actions from the staged probabilities and copies the outputs to global memory, for both
// buffers in tile order, while the MMA warpgroups go on to their next tile.  Each staging
// buffer is single-buffered between a full / empty mbarrier pair: the MMA warpgroup waits on
// `empty` only when it is about to stage its next tile, a whole tile of MMAs later.  (The
// softmax stays with the MMA warpgroups: measured with WDB_PHASE_CLOCKS, one warpgroup doing
// the softmax too for both halves of a tile took longer than the tile's MMAs.)
// Registers: the CTA starts at 168 per thread (65536 / 384, in steps of 8) and setmaxnreg
// moves them between the roles.  A warpgroup can only grow by what the CTA's other warpgroups
// released, so 2 x kMmaRegs + kEpiRegs must not exceed 3 x 168 (more and the MMA warpgroups
// would wait for registers forever).
constexpr int kSampledThreads = kThreads + 128;
constexpr int kSampledLaunchRegs = (65536 / kSampledThreads) & ~7;
// (ptxas 12.9: neither role spills)
constexpr int kMmaRegs = 224, kEpiRegs = 56;
static_assert(kWarpgroups * kMmaRegs + kEpiRegs <= (kWarpgroups + 1) * kSampledLaunchRegs,
              "setmaxnreg can only hand out the registers the CTA was launched with");
// named barrier of the epilogue warpgroup (1 and 2 are the MMA warpgroups' wg_sync)
__device__ __forceinline__ void epi_sync() { asm volatile("bar.sync 3, 128;" ::: "memory"); }
__device__ __forceinline__ void mbar_arrive(uint32_t mbar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(mbar) : "memory");
}
// shared memory: weights | a staging buffer per MMA warpgroup (its logits, then the epilogue's
// outputs) | mbarriers: weights landed, full[2], empty[2]
constexpr int kSampledStageBytes = kWgRows * FastShape::N3 * 4;
constexpr int kSampledBarriers = 1 + 2 * kWarpgroups;

// Profiling aid (-DWDB_PHASE_CLOCKS): like mlp_forward_body's, but per tile k < 18 of the CTA
// [3 + 5 k + p]: p = 0 tile start (warpgroup 0), 1 warpgroup 0's layer 1 done, 2 warpgroup 0's
// MMAs done, 3 warpgroup 1's MMAs done, 4 the epilogue warpgroup has stored both halves.
template <bool TILES>
__global__ void __launch_bounds__(kSampledThreads, 1)
mlp_forward_sampled_kernel(const unsigned char *__restrict__ blob, const void *__restrict__ input,
                           long long rows, float *__restrict__ probs0, float *__restrict__ probs1,
                           float *__restrict__ values, const __grid_constant__ MlpSampling smp) {
  using Shape = FastShape;
  extern __shared__ __align__(128) unsigned char smem[];
  const MlpHeader hd = *reinterpret_cast<const MlpHeader *>(blob);
  const int F = hd.F, A0 = hd.A0, A1 = hd.A1;
  constexpr int N3 = Shape::N3;
  constexpr MlpLayout lay = mlp_layout(Shape::K1, Shape::H, Shape::N3);
  constexpr int w_bytes = lay.total_bytes - lay.off_w1;  // W1 | W2 | W3 | biases, contiguous
  unsigned char *s_w = smem;
  const uint32_t s_w1 = smem_addr(s_w);
  const uint32_t s_w2 = s_w1 + (lay.off_w2 - lay.off_w1);
  const uint32_t s_w3 = s_w1 + (lay.off_w3 - lay.off_w1);
  const float *s_b1 = reinterpret_cast<const float *>(s_w + (lay.off_b - lay.off_w1));
  const float *s_b2 = s_b1 + Shape::H;
  const float *s_b3 = s_b2 + Shape::H;
  constexpr int stage0 = (w_bytes + 127) & ~127;
  const uint32_t bar_w = smem_addr(s_w + stage0 + kWarpgroups * kSampledStageBytes);
  auto bar_full = [&](int w) { return bar_w + 8 * (1 + w); };
  auto bar_empty = [&](int w) { return bar_w + 8 * (1 + kWarpgroups + w); };
  auto stage = [&](int w) { return reinterpret_cast<float *>(s_w + stage0 + w * kSampledStageBytes); };
  const int tid = threadIdx.x, lt = tid & 127, wg = tid >> 7;
  const unsigned bid = blockIdx.x, gdim = gridDim.x;
  const long long n_tiles = (rows + kTileM - 1) / kTileM;
#ifdef WDB_PHASE_CLOCKS
  __shared__ int s_rec;
  if (tid == 0) {
    s_rec = bid == 0 && atomicCAS(&g_mlp_clocks_busy, 0, 1) == 0;
    if (s_rec) {
      for (int i = 0; i < kMlpClockSlots; i++) g_mlp_clocks[i] = 0;
      g_mlp_clocks[0] = rows;
    }
  }
  __syncthreads();
  const bool rec_clocks = s_rec && lt == 0;
  int clock_tile = 0;
#endif
  if (tid == 0) MLP_MARK(1);
  if (tid == 0) {
    mbar_init(bar_w, 1);
    for (int w = 0; w < kWarpgroups; w++) {
      mbar_init(bar_full(w), 128);
      mbar_init(bar_empty(w), 128);
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  // (the PDL order of mlp_forward_body with flags = 0: the weights are read after the wait)
  griddep_wait();
  if (tid == 0) {                                         // weights: TMA bulk copies
    mbar_expect_tx(bar_w, (uint32_t)w_bytes);
    uint32_t off = 0;
    while (off < (uint32_t)w_bytes) {
      const uint32_t n = min((uint32_t)w_bytes - off, 65536u);
      tma_load(s_w1 + off, blob + lay.off_w1 + off, n, bar_w);
      off += n;
    }
  }
  griddep_launch_dependents();

  if (wg < kWarpgroups) {
    // ---- MMA warpgroup wg: rows [tile * 128 + 64 wg, + 64) of each of the CTA's tiles
    asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(kMmaRegs));
    ObsFrag<TILES, Shape::K1> next;
    uint32_t a1[Shape::K1 / 4];
    const bool have_first = bid < n_tiles && bid * kTileM + wg * kWgRows < rows;
    if (have_first) obs_frag_load(next, 0, input, rows, F, bid * kTileM + wg * kWgRows);
    mbar_wait(bar_w, 0);
    if (tid == 0) MLP_MARK(2);
    if (have_first) {
      obs_frag_pack(next, 0, a1);
      obs_frag_load(next, 1, input, rows, F, bid * kTileM + wg * kWgRows);
      obs_frag_pack(next, 1, a1);
    }
    constexpr uint32_t sbo_a = (uint32_t)(Shape::K1 / 8) * 128u;
    constexpr uint32_t sbo_h = (uint32_t)(Shape::H / 8) * 128u;
    const int lane = tid & 31, lr = ((tid >> 5) & 3) * 16 + (lane >> 2), t = lane & 3;
    uint32_t phase = 1;          // an empty buffer: the wait on the phase before the first passes
    for (long long tile = bid; tile < n_tiles; tile += gdim) {
      const long long row0 = tile * kTileM + wg * kWgRows;
      if (row0 >= rows) break;   // (warpgroup-uniform; so are all later tiles)
#ifdef WDB_PHASE_CLOCKS
      const int mark0 = 3 + 5 * (clock_tile < 18 ? clock_tile : kMlpClockSlots);
      clock_tile++;
#endif
      if (wg == 0) MLP_MARK(mark0);
      uint32_t h[kMaxK / 4];
      fast_layer1(a1, s_w1, sbo_a, s_b1, h);
      if (wg == 0) MLP_MARK(mark0 + 1);
      float o[kMaxN3 / 16][8];
      float(&o48)[48 / 2] = *reinterpret_cast<float(*)[48 / 2]>(&o[0][0]);
      fast_layers23<TILES>(h, s_w2, s_w3, sbo_h, s_b2, o48, next, a1,
                           row0 + (long long)gdim * kTileM < rows, input, rows, F,
                           row0 + (long long)gdim * kTileM);
      wgmma_wait<0>();
      MLP_MARK(mark0 + 2 + wg);
      mbar_wait(bar_empty(wg), phase);      // the epilogue has copied out the previous tile
      phase ^= 1;
      float *s_o = stage(wg);
      stage_logits(o, s_b3, N3, lr, t, s_o);
      wg_sync(wg);
      // thread lt: row lt % 64; lt < 64 head 0, else head 1 + the value (mlp_forward_body's
      // softmax).  (Derived from an opaque copy of lt: otherwise they, and the 32
      // staged-logit addresses, are hoisted out of the tile loop and held across its MMAs.)
      int l = lt;
      asm volatile("" : "+r"(l));
      const int row = l & 63, part = l >> 6;
      const int cbase = part ? A0 : 0, cnt = part ? A1 : A0;
      float lg[32], value;
      const float inv = softmax_row(s_o, N3, row, cbase, cnt, lg, value);
      wg_sync(wg);                          // every logit has been read
      float *dst = s_o + (part ? kWgRows * A0 : 0) + row * cnt;
#pragma unroll
      for (int i = 0; i < 32; i++)
        if (i < cnt) dst[i] = lg[i] * inv;
      if (part) s_o[kWgRows * (A0 + A1) + row] = value;
      mbar_arrive(bar_full(wg));
    }
  } else {
    // ---- epilogue warpgroup: thread lt samples head lt / 64 of row lt % 64 of each staged
    // half-tile, in tile order, and the warpgroup copies the half-tile's outputs out
    asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(kEpiRegs));
    const int row = lt & 63, part = lt >> 6;
    const int cnt = part ? A1 : A0;
    uint32_t phase = 0;
    for (long long tile = bid; tile < n_tiles; tile += gdim) {
#ifdef WDB_PHASE_CLOCKS
      const int mark0 = 3 + 5 * (clock_tile < 18 ? clock_tile : kMlpClockSlots);
      clock_tile++;
#endif
#pragma unroll 1
      for (int w = 0; w < kWarpgroups; w++) {
        const long long rb = tile * kTileM + w * kWgRows;   // first row of the half-tile
        if (rb >= rows) break;
        // this thread's uniform's inputs, requested before the wait so that the loads overlap
        // it; both threads of a row read the RNG offset before the epi_sync below, the head-0
        // thread advances it after that barrier
        const long long s_row = rb + row;
        const bool s_valid = s_row < rows;
        long long s_gi = 0;
        unsigned long long s_seed = 0, s_off = 0;
        float s_u = 0.0f;
        if (s_valid) {
          const long long prow = smp.row0 + s_row;          // row of the policy
          const long long env = prow / smp.Np;
          s_gi = env * smp.N + __ldg(smp.agent + (int)(prow - env * smp.Np));
          if (smp.uniforms) {
            s_u = __ldg(smp.uniforms + 2 * s_gi + part);
          } else {
            s_seed = reinterpret_cast<const RngHeader *>(smp.rng)->seed;
            s_off = rng_offsets(smp.rng)[s_gi];
          }
        }
        const float *s_o = stage(w);
        mbar_wait(bar_full(w), phase);
        epi_sync();
        if (s_valid) {
          if (!smp.uniforms) {
            RngHeader h;
            h.seed = s_seed; h.n_streams = 0;
            const uint4 d = rng_draw4(h, (unsigned long long)s_gi, s_off);
            s_u = u32_to_uniform(part ? d.y : d.x);
            if (!part) rng_offsets(smp.rng)[s_gi] = s_off + 1;
          }
          // the probabilities exactly as they were stored, sampled in registers
          const float *src = s_o + (part ? kWgRows * A0 : 0) + row * cnt;
          float p[32];
#pragma unroll
          for (int i = 0; i < 32; i++) p[i] = i < cnt ? src[i] : 0.0f;
          smp.actions[2 * s_row + part] = sample_cdf_regs(p, cnt, s_u);
        }
        copy_outputs(s_o, rb, rows, A0, A1, probs0, probs1, values, lt);
        mbar_arrive(bar_empty(w));                           // the buffer may be restaged
      }
      phase ^= 1;
      MLP_MARK(mark0 + 4);
    }
  }
#ifdef WDB_PHASE_CLOCKS
  __syncthreads();
  if (tid == 0 && s_rec) {
    __threadfence();
    atomicExch(&g_mlp_clocks_busy, 0);
  }
#endif
}

template <class Shape>
__global__ void __launch_bounds__(kThreads, 1)
mlp_forward_masked_kernel(const unsigned char *__restrict__ blob, const float *__restrict__ obs,
                          long long rows, const float *__restrict__ mask,
                          float *__restrict__ probs0, float *__restrict__ probs1,
                          float *__restrict__ values) {
  mlp_forward_body<false, Shape, true>(blob, obs, rows, probs0, probs1, values, blockIdx.x,
                                       gridDim.x, 0, mask);
}

// Two policies in ONE grid: CTAs [0, split) run policy A, the rest policy B (each persistent
// over its own tiles).  Replaces the fork / join of two launches on two streams.
struct MlpPairArgs {
  const unsigned char *blob[2];
  const float *obs[2];
  long long rows[2];
  float *probs0[2], *probs1[2], *values[2];
  unsigned split;
  int flags;
};
__global__ void __launch_bounds__(kThreads, 1)
mlp_forward_pair_kernel(const __grid_constant__ MlpPairArgs a) {
  const int w = blockIdx.x >= a.split ? 1 : 0;
  mlp_forward_body<false, AnyShape>(a.blob[w], a.obs[w], a.rows[w], a.probs0[w], a.probs1[w],
                                    a.values[w], w ? blockIdx.x - a.split : blockIdx.x,
                                    w ? gridDim.x - a.split : a.split, a.flags);
}

// ---- weight packing: fp32 nn.Linear weights [out, in] -> bf16 canonical K-major tiles ------
__global__ void pack_matrix_kernel(const float *__restrict__ w, int n_rows, int n_cols,
                                   int n_pad, int k_pad, __nv_bfloat16 *__restrict__ out) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;    // over n_pad * k_pad
  if (i >= n_pad * k_pad) return;
  const int n = i / k_pad, k = i - n * k_pad;
  const float v = (n < n_rows && k < n_cols) ? w[(long long)n * n_cols + k] : 0.0f;
  const int off = (n >> 3) * (k_pad / 8) * 64 + (k >> 3) * 64 + (n & 7) * 8 + (k & 7);
  out[off] = __float2bfloat16_rn(v);
}

__global__ void pack_rows_kernel(const float *__restrict__ w, int rows, int n_cols, int row0,
                                 int k_pad, __nv_bfloat16 *__restrict__ out) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= rows * n_cols) return;
  const int rr = i / n_cols, k = i - rr * n_cols;
  const int n = row0 + rr;
  const int off = (n >> 3) * (k_pad / 8) * 64 + (k >> 3) * 64 + (n & 7) * 8 + (k & 7);
  out[off] = __float2bfloat16_rn(w[i]);
}

__global__ void pack_misc_kernel(MlpHeader hd, unsigned char *blob, const float *b1,
                                 const float *b2, const float *bh0, const float *bh1,
                                 const float *bv) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i == 0) *reinterpret_cast<MlpHeader *>(blob) = hd;
  float *b = reinterpret_cast<float *>(blob + hd.off_b);
  if (i < hd.H) { b[i] = b1[i]; b[hd.H + i] = b2[i]; }
  if (i < hd.N3) {
    float v = 0.0f;
    if (i < hd.A0) v = bh0[i];
    else if (i < hd.A0 + hd.A1) v = bh1[i - hd.A0];
    else if (i == hd.A0 + hd.A1) v = bv[0];
    b[2 * hd.H + i] = v;
  }
}

MlpHeader make_header(int F, int H, int A0, int A1) {
  MlpHeader hd;
  hd.F = F; hd.K1 = round_up(F, 16); hd.H = H; hd.A0 = A0; hd.A1 = A1;
  hd.N3 = round_up(A0 + A1 + 1, 16);
  const MlpLayout l = mlp_layout(hd.K1, H, hd.N3);
  hd.off_w1 = l.off_w1;
  hd.off_w2 = l.off_w2;
  hd.off_w3 = l.off_w3;
  hd.off_b = l.off_b;
  hd.total_bytes = l.total_bytes;
  hd.pad = 0;
  return hd;
}

size_t mlp_smem_bytes(const MlpHeader &hd) {
  const size_t w = (size_t)hd.total_bytes - hd.off_w1;
  const size_t stage = (size_t)kWgRows * max(hd.K1 * 2, hd.N3 * 4);
  return ((w + 127) & ~(size_t)127) + kWarpgroups * stage + 16;   // + the weights' mbarrier
}

bool mlp_shape_ok(int F, int H, int A0, int A1) {
  // A1 == 0: a single-head policy (gridworld, classic control); the second output part then
  // carries only the value column
  return F >= 1 && F <= 256 && H >= 16 && H <= 256 && (H % 32) == 0 && A0 >= 1 && A1 >= 0 &&
         A0 <= 32 && A1 + 1 <= 32;
}

}  // namespace

// wdb_set_option("mlp_max_ctas", n): CTAs (= SMs, one persistent CTA each) the NEXT forward
// launches may use; 0 = all.  Lets two policies' forwards run side by side on disjoint SMs.
int g_mlp_max_ctas = 0;
namespace wdb {
int g_pdl = 0;            // wdb_set_option("pdl", 0/1): programmatic dependent launches (A/B: slower)
}

WDB_API long long wdb_mlp_blob_bytes(int F, int H, int A0, int A1) {
  if (!mlp_shape_ok(F, H, A0, A1)) return -1;
  const MlpHeader hd = make_header(F, H, A0, A1);
  if (mlp_smem_bytes(hd) > 227 * 1024) return -1;
  return hd.total_bytes;
}

WDB_API int wdb_mlp_pack_weights(void *stream, void *blob, const float *w1, const float *b1,
                                 const float *w2, const float *b2, const float *wh0,
                                 const float *bh0, const float *wh1, const float *bh1,
                                 const float *wv, const float *bv, int F, int H, int A0,
                                 int A1) {
  if (!blob || !w1 || !b1 || !w2 || !b2 || !wh0 || !bh0 || !wv || !bv)
    return (int)cudaErrorInvalidValue;
  if (A1 > 0 && (!wh1 || !bh1)) return (int)cudaErrorInvalidValue;
  if (!mlp_shape_ok(F, H, A0, A1)) return (int)cudaErrorInvalidValue;
  const MlpHeader hd = make_header(F, H, A0, A1);
  cudaStream_t st = as_stream(stream);
  unsigned char *b = reinterpret_cast<unsigned char *>(blob);
  auto bf = [&](int off) { return reinterpret_cast<__nv_bfloat16 *>(b + off); };
  cudaError_t e = cudaMemsetAsync(b + hd.off_w3, 0, (size_t)hd.N3 * H * 2, st);
  if (e != cudaSuccess) return (int)e;
  const int T = 256;
  pack_matrix_kernel<<<(H * hd.K1 + T - 1) / T, T, 0, st>>>(w1, H, F, H, hd.K1, bf(hd.off_w1));
  pack_matrix_kernel<<<(H * H + T - 1) / T, T, 0, st>>>(w2, H, H, H, H, bf(hd.off_w2));
  // W3 = [head0; head1; value] stacked along N (zero padded to N3 rows by the memset)
  pack_rows_kernel<<<(A0 * H + T - 1) / T, T, 0, st>>>(wh0, A0, H, 0, H, bf(hd.off_w3));
  if (A1 > 0)
    pack_rows_kernel<<<(A1 * H + T - 1) / T, T, 0, st>>>(wh1, A1, H, A0, H, bf(hd.off_w3));
  pack_rows_kernel<<<(H + T - 1) / T, T, 0, st>>>(wv, 1, H, A0 + A1, H, bf(hd.off_w3));
  g_launch_count += 5;
  pack_misc_kernel<<<(max(H, hd.N3) + T - 1) / T, T, 0, st>>>(hd, b, b1, b2, bh0, bh1, bv);
  return finish_launch();
}

namespace {

// mask != NULL (fp32 observations only): the masked kernel
template <bool TILES, class Shape>
int launch_forward_shape(cudaStream_t stream, const void *blob, size_t smem, const void *input,
                         long long rows, const float *mask, float *probs0, float *probs1,
                         float *values) {
  static size_t configured = 0, configured_masked = 0;
  size_t &conf = mask ? configured_masked : configured;
  if (smem > conf) {
    cudaError_t e = mask ? cudaFuncSetAttribute(mlp_forward_masked_kernel<Shape>,
                                                cudaFuncAttributeMaxDynamicSharedMemorySize,
                                                (int)smem)
                         : cudaFuncSetAttribute(mlp_forward_kernel<TILES, Shape>,
                                                cudaFuncAttributeMaxDynamicSharedMemorySize,
                                                (int)smem);
    if (e != cudaSuccess) return (int)e;
    conf = smem;
  }
  const long long n_tiles = (rows + kTileM - 1) / kTileM;
  const int sm_budget = (g_mlp_max_ctas > 0 && g_mlp_max_ctas < kNumSMs) ? g_mlp_max_ctas : kNumSMs;
  const int grid = (int)min((long long)sm_budget, n_tiles);
  if (mask)
    mlp_forward_masked_kernel<Shape><<<grid, kThreads, smem, stream>>>(
        reinterpret_cast<const unsigned char *>(blob), reinterpret_cast<const float *>(input),
        rows, mask, probs0, probs1, values);
  else
    mlp_forward_kernel<TILES, Shape><<<grid, kThreads, smem, stream>>>(
        reinterpret_cast<const unsigned char *>(blob), input, rows, probs0, probs1, values, 0);
  return finish_launch();
}

template <bool TILES>
int launch_forward(void *stream, const void *blob, int F, int H, int A0, int A1,
                   const void *input, long long rows, float *probs0, float *probs1,
                   float *values, const float *mask = nullptr) {
  if (!blob || !input || !probs0 || (A1 > 0 && !probs1) || rows <= 0)
    return (int)cudaErrorInvalidValue;
  if (TILES && mask) return (int)cudaErrorInvalidValue;
  if (!mlp_shape_ok(F, H, A0, A1)) return (int)cudaErrorInvalidValue;
  if (TILES && (reinterpret_cast<uintptr_t>(input) & 15)) return (int)cudaErrorInvalidValue;
  const MlpHeader hd = make_header(F, H, A0, A1);
  const size_t smem = mlp_smem_bytes(hd);
  if (smem > 227 * 1024) return (int)cudaErrorInvalidValue;
  const bool fast = hd.K1 == FastShape::K1 && hd.H == FastShape::H && hd.N3 == FastShape::N3;
  return (fast ? launch_forward_shape<TILES, FastShape> : launch_forward_shape<TILES, AnyShape>)(
      as_stream(stream), blob, smem, input, rows, mask, probs0, probs1, values);
}

bool mlp_samples(int F, int H, int A0, int A1) {
  if (!mlp_shape_ok(F, H, A0, A1) || A1 < 1) return false;
  const MlpHeader hd = make_header(F, H, A0, A1);
  return hd.K1 == FastShape::K1 && hd.H == FastShape::H && hd.N3 == FastShape::N3;
}

template <bool TILES>
int launch_forward_sampled(void *stream, const void *blob, int F, int H, int A0, int A1,
                           const void *input, long long rows, float *probs0, float *probs1,
                           float *values, const wdb_mlp_sampling *s) {
  if (!blob || !input || !probs0 || !probs1 || rows <= 0 || !s) return (int)cudaErrorInvalidValue;
  if (!mlp_samples(F, H, A0, A1)) return (int)cudaErrorInvalidValue;
  if (TILES && (reinterpret_cast<uintptr_t>(input) & 15)) return (int)cudaErrorInvalidValue;
  if (!s->actions || !s->agent_of_slot || (!s->rng_state && !s->uniforms))
    return (int)cudaErrorInvalidValue;
  if (reinterpret_cast<uintptr_t>(s->actions) & 7) return (int)cudaErrorMisalignedAddress;
  if (s->n_policy_agents < 1 || s->n_agents < s->n_policy_agents || rows % s->n_policy_agents)
    return (int)cudaErrorInvalidValue;
  if (s->row_offset < 0 || s->row_offset % s->n_policy_agents) return (int)cudaErrorInvalidValue;
  constexpr MlpLayout lay = mlp_layout(FastShape::K1, FastShape::H, FastShape::N3);
  const size_t smem = (size_t)((lay.total_bytes - lay.off_w1 + 127) & ~127) +
                      kWarpgroups * kSampledStageBytes + 8 * kSampledBarriers;
  static size_t configured = 0;
  if (smem > configured) {
    const cudaError_t e = cudaFuncSetAttribute(mlp_forward_sampled_kernel<TILES>,
                                               cudaFuncAttributeMaxDynamicSharedMemorySize,
                                               (int)smem);
    if (e != cudaSuccess) return (int)e;
    configured = smem;
  }
  const MlpSampling smp = {s->actions, s->rng_state, s->uniforms, s->agent_of_slot, s->n_agents,
                           s->n_policy_agents, s->row_offset};
  const long long n_tiles = (rows + kTileM - 1) / kTileM;
  const int sm_budget = (g_mlp_max_ctas > 0 && g_mlp_max_ctas < kNumSMs) ? g_mlp_max_ctas : kNumSMs;
  const int grid = (int)min((long long)sm_budget, n_tiles);
  mlp_forward_sampled_kernel<TILES><<<grid, kSampledThreads, smem, as_stream(stream)>>>(
      reinterpret_cast<const unsigned char *>(blob), input, rows, probs0, probs1, values, smp);
  return finish_launch();
}

// Launch with the programmatic-stream-serialization attribute when the "pdl" option is on:
// the grid may start while the previous kernel of the stream drains; the kernels order
// themselves with griddepcontrol.wait (under stream capture this becomes a programmatic edge
// of the CUDA graph).
int launch_forward_pair(void *stream, const wdb_mlp_pair &p) {
  MlpPairArgs a = {};
  size_t smem = 0;
  long long tiles[2];
  for (int w = 0; w < 2; w++) {
    if (!p.blob[w] || !p.obs[w] || !p.probs0[w] || (p.A1[w] > 0 && !p.probs1[w]) || p.rows[w] <= 0)
      return (int)cudaErrorInvalidValue;
    if (!mlp_shape_ok(p.F[w], p.H[w], p.A0[w], p.A1[w])) return (int)cudaErrorInvalidValue;
    const MlpHeader hd = make_header(p.F[w], p.H[w], p.A0[w], p.A1[w]);
    const size_t need = mlp_smem_bytes(hd);
    if (need > smem) smem = need;
    a.blob[w] = reinterpret_cast<const unsigned char *>(p.blob[w]);
    a.obs[w] = p.obs[w];
    a.rows[w] = p.rows[w];
    a.probs0[w] = p.probs0[w]; a.probs1[w] = p.probs1[w]; a.values[w] = p.values[w];
    tiles[w] = (p.rows[w] + kTileM - 1) / kTileM;
  }
  if (smem > 227 * 1024) return (int)cudaErrorInvalidValue;
  static size_t configured = 0;
  if (smem > configured) {
    cudaError_t e = cudaFuncSetAttribute(mlp_forward_pair_kernel,
                                         cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return (int)e;
    configured = smem;
  }
  int cb = p.ctas_b;
  if (cb <= 0) {
    // cost in tile-times: the slower of the two shares (the smaller share's tiles run ~1.3x
    // slower: fewer CTAs keep its weights hot in L2)
    double best = 1e30;
    for (int k = 1; k < kNumSMs; k++) {
      const double ca = (double)((tiles[0] + kNumSMs - k - 1) / (kNumSMs - k));
      const double cbt = (double)((tiles[1] + k - 1) / k);
      const double cost = tiles[0] >= tiles[1] ? fmax(ca, 1.3 * cbt) : fmax(1.3 * ca, cbt);
      if (cost < best) { best = cost; cb = k; }
    }
  }
  if (cb >= kNumSMs) cb = kNumSMs - 1;
  long long ca = kNumSMs - cb;
  if (ca > tiles[0]) ca = tiles[0];
  if (cb > tiles[1]) cb = (int)tiles[1];
  a.split = (unsigned)ca;
  a.flags = p.flags;
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3((unsigned)(ca + cb), 1, 1);
  cfg.blockDim = dim3(kThreads, 1, 1);
  cfg.dynamicSmemBytes = smem;
  cfg.stream = as_stream(stream);
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = g_pdl ? 1 : 0;
  const cudaError_t e = cudaLaunchKernelEx(&cfg, mlp_forward_pair_kernel, a);
  if (e != cudaSuccess) return (int)e;
  return finish_launch();
}

// fp32 obs [rows, F] -> bf16 A-operand tiles (128 rows x K1, canonical K-major layout, K
// padding and the rows of the last tile beyond `rows` = 0): one thread per 16-byte chunk
__global__ void pack_obs_kernel(const float *__restrict__ obs, long long rows, int F, int K1,
                                unsigned char *__restrict__ tiles) {
  const int nchunk = K1 / 8;
  const long long n_tiles = (rows + kTileM - 1) / kTileM;
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_tiles * kTileM * nchunk) return;
  // consecutive threads: the 8 rows of a core matrix, then the next chunk of the same rows
  const long long grp = i / (8 * nchunk);                 // 8-row group (global)
  const int in = (int)(i - grp * 8 * nchunk);
  const int c = in >> 3, rr = in & 7;
  const long long row = grp * 8 + rr;
  float v[8];
#pragma unroll
  for (int k = 0; k < 8; k++)
    v[k] = (row < rows && 8 * c + k < F) ? obs[row * F + 8 * c + k] : 0.0f;
  uint4 o;
  o.x = pack_bf16(v[0], v[1]); o.y = pack_bf16(v[2], v[3]); o.z = pack_bf16(v[4], v[5]); o.w = pack_bf16(v[6], v[7]);
  const long long t = row >> 7;
  const int r = (int)(row & 127);
  *reinterpret_cast<uint4 *>(tiles + t * ((long long)kTileM * K1 * 2) + (r >> 3) * (K1 * 16) +
                             c * 128 + (r & 7) * 16) = o;
}

}  // namespace

WDB_API long long wdb_mlp_obs_tiles_bytes(int F, long long rows) {
  if (F < 1 || F > 256 || rows <= 0) return -1;
  const long long n_tiles = (rows + kTileM - 1) / kTileM;
  return n_tiles * kTileM * round_up(F, 16) * 2;
}

WDB_API int wdb_mlp_pack_obs(void *stream, const float *obs, long long rows, int F,
                             void *tiles) {
  if (!obs || !tiles || rows <= 0 || F < 1 || F > 256) return (int)cudaErrorInvalidValue;
  const int K1 = round_up(F, 16);
  const long long n = ((rows + kTileM - 1) / kTileM) * kTileM * (K1 / 8);
  const int T = 256;
  pack_obs_kernel<<<(unsigned)((n + T - 1) / T), T, 0, as_stream(stream)>>>(
      obs, rows, F, K1, reinterpret_cast<unsigned char *>(tiles));
  return finish_launch();
}

WDB_API int wdb_mlp_policy_forward(void *stream, const void *blob, int F, int H, int A0, int A1,
                                   const float *obs, long long rows, float *probs0,
                                   float *probs1, float *values) {
  return launch_forward<false>(stream, blob, F, H, A0, A1, obs, rows, probs0, probs1, values);
}

WDB_API int wdb_mlp_policy_forward_masked(void *stream, const void *blob, int F, int H, int A0,
                                          int A1, const float *obs, long long rows,
                                          const float *mask, float *probs0, float *probs1,
                                          float *values) {
  if (!mask) return (int)cudaErrorInvalidValue;
  return launch_forward<false>(stream, blob, F, H, A0, A1, obs, rows, probs0, probs1, values,
                               mask);
}

WDB_API int wdb_mlp_forward_samples(int F, int H, int A0, int A1) {
  return mlp_samples(F, H, A0, A1) ? 1 : 0;
}

WDB_API int wdb_mlp_policy_forward_sampled(void *stream, const void *blob, int F, int H, int A0,
                                           int A1, const void *input, int input_is_tiles,
                                           long long rows, float *probs0, float *probs1,
                                           float *values, const wdb_mlp_sampling *sampling) {
  return (input_is_tiles ? launch_forward_sampled<true> : launch_forward_sampled<false>)(
      stream, blob, F, H, A0, A1, input, rows, probs0, probs1, values, sampling);
}

WDB_API int wdb_mlp_policy_forward_pair(void *stream, const wdb_mlp_pair *pair) {
  if (!pair) return (int)cudaErrorInvalidValue;
  return launch_forward_pair(stream, *pair);
}

#ifdef WDB_PHASE_CLOCKS
// the phase clocks of the last recorded forward launch (see MLP_MARK)
WDB_API int wdb_debug_mlp_clocks(long long *out) {
  if (!out) return (int)cudaErrorInvalidValue;
  return (int)cudaMemcpyFromSymbol(out, g_mlp_clocks, sizeof(g_mlp_clocks));
}
#endif

WDB_API int wdb_mlp_policy_forward_tiles(void *stream, const void *blob, int F, int H, int A0,
                                         int A1, const void *obs_tiles, long long rows,
                                         float *probs0, float *probs1, float *values) {
  return launch_forward<true>(stream, blob, F, H, A0, A1, obs_tiles, rows, probs0, probs1,
                              values);
}
