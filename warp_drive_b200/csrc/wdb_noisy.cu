// wdb_noisy.cu -- the noisy head's noise draws, its effective layers and the map of their
// gradients onto mu and sigma (include/wdb200.h, wdb_noisy_*).
//
// A noisy DQN or C51 update runs the unchanged pass on the effective layers: materialize writes
// them (and the f(eps) vectors) from mu, sigma and the update's noise before the pass, and the
// grads launch maps the pass's gradients of the effective layers onto mu and sigma after it.
// Acting draws per-row noise with wdb_noisy_draw.  Each launch computes one element per thread
// with no sums, so all three are bit-reproducible; every noise value comes from noisy_f.
#include "wdb_noisy.cuh"

using namespace wdb;

namespace {

constexpr int kThreads = 256;
constexpr long long kMaxBlocks = 4096;

// Finds the layer of element i of a per-layer sequence of `size(layer)` elements; i becomes
// the index within that layer.  -1 past the end.
template <typename Size>
__device__ __forceinline__ int layer_of(const wdb_noisy_net &n, long long &i, Size size) {
  for (int l = 0; l < n.n_layers; ++l) {
    const long long s = size(n.layer[l]);
    if (i < s) return l;
    i -= s;
  }
  return -1;
}

__device__ __forceinline__ long long noise_size(const wdb_noisy_layer &L) {
  return (long long)L.in_dim + L.out_dim;
}

__device__ __forceinline__ long long layer_size(const wdb_noisy_layer &L) {
  return (long long)L.out_dim * L.in_dim + L.out_dim;
}

__host__ __device__ inline long long total(const wdb_noisy_net &n, bool with_noise) {
  long long t = 0;
  for (int l = 0; l < n.n_layers; ++l) {
    const wdb_noisy_layer &L = n.layer[l];
    t += (long long)L.out_dim * L.in_dim + L.out_dim + (with_noise ? L.in_dim + L.out_dim : 0);
  }
  return t;
}

__global__ void __launch_bounds__(kThreads)
noisy_draw_kernel(wdb_noisy_net net, unsigned long long seed, int domain,
                  unsigned long long count, int row0, int n_rows) {
  long long per_row = 0;
  for (int l = 0; l < net.n_layers; ++l) per_row += noise_size(net.layer[l]);
  const long long all = per_row * n_rows;
  for (long long i = (long long)blockIdx.x * kThreads + threadIdx.x; i < all;
       i += (long long)gridDim.x * kThreads) {
    const long long r = i / per_row;
    long long e = i % per_row;
    const int l = layer_of(net, e, noise_size);
    const wdb_noisy_layer &L = net.layer[l];
    const float v = noisy_f(seed, domain, count, (uint32_t)(row0 + r), l, (int)e);
    if (e < L.in_dim) L.noise_in[r * L.in_dim + e] = v;
    else L.noise_out[r * L.out_dim + (e - L.in_dim)] = v;
  }
}

// Per layer: the in + out noise elements, then W [out, in], then b [out].
__global__ void __launch_bounds__(kThreads)
noisy_materialize_kernel(wdb_noisy_net online, wdb_noisy_net target, unsigned long long seed,
                         unsigned long long update) {
  const wdb_noisy_net &net = blockIdx.y == 0 ? online : target;
  const uint32_t row = blockIdx.y;
  const long long all = total(net, true);
  for (long long i = (long long)blockIdx.x * kThreads + threadIdx.x; i < all;
       i += (long long)gridDim.x * kThreads) {
    long long e = i;
    const int l = layer_of(net, e, [](const wdb_noisy_layer &L) {
      return noise_size(L) + layer_size(L);
    });
    const wdb_noisy_layer &L = net.layer[l];
    const int in = L.in_dim, out = L.out_dim;
    if (e < in + out) {
      const float v = noisy_f(seed, 0, update, row, l, (int)e);
      if (e < in) L.noise_in[e] = v;
      else L.noise_out[e - in] = v;
      continue;
    }
    e -= in + out;
    if (e < (long long)out * in) {
      const int j = (int)(e / in), k = (int)(e % in);
      const float fo = noisy_f(seed, 0, update, row, l, in + j);
      const float fi = noisy_f(seed, 0, update, row, l, k);
      L.weight[e] = __fmaf_rn(L.weight_sigma[e], __fmul_rn(fo, fi), L.weight_mu[e]);
    } else {
      const int j = (int)(e - (long long)out * in);
      const float fo = noisy_f(seed, 0, update, row, l, in + j);
      L.bias[j] = __fmaf_rn(L.bias_sigma[j], fo, L.bias_mu[j]);
    }
  }
}

__global__ void __launch_bounds__(kThreads) noisy_grads_kernel(wdb_noisy_net net) {
  const long long all = total(net, false);
  for (long long i = (long long)blockIdx.x * kThreads + threadIdx.x; i < all;
       i += (long long)gridDim.x * kThreads) {
    long long e = i;
    const int l = layer_of(net, e, layer_size);
    const wdb_noisy_layer &L = net.layer[l];
    const int in = L.in_dim, out = L.out_dim;
    if (e < (long long)out * in) {
      const int j = (int)(e / in), k = (int)(e % in);
      const float g = L.grad_weight[e];
      L.grad_weight_mu[e] = g;
      L.grad_weight_sigma[e] = __fmul_rn(g, __fmul_rn(L.noise_out[j], L.noise_in[k]));
    } else {
      const int j = (int)(e - (long long)out * in);
      const float g = L.grad_bias[j];
      L.grad_bias_mu[j] = g;
      L.grad_bias_sigma[j] = __fmul_rn(g, L.noise_out[j]);
    }
  }
}

bool shape_ok(const wdb_noisy_net *n) {
  if (!n || n->n_layers < 1 || n->n_layers > WDB_NOISY_MAX_LAYERS) return false;
  for (int l = 0; l < n->n_layers; ++l) {
    const wdb_noisy_layer &L = n->layer[l];
    if (L.in_dim < 1 || L.out_dim < 1 || (long long)L.in_dim + L.out_dim > (1ll << 17))
      return false;
    if ((long long)L.in_dim * L.out_dim >= (1ll << 31)) return false;
  }
  return true;
}

bool same_shape(const wdb_noisy_net &a, const wdb_noisy_net &b) {
  if (a.n_layers != b.n_layers) return false;
  for (int l = 0; l < a.n_layers; ++l)
    if (a.layer[l].in_dim != b.layer[l].in_dim || a.layer[l].out_dim != b.layer[l].out_dim)
      return false;
  return true;
}

bool materialize_pointers_ok(const wdb_noisy_net &n) {
  for (int l = 0; l < n.n_layers; ++l) {
    const wdb_noisy_layer &L = n.layer[l];
    if (!L.weight_mu || !L.weight_sigma || !L.bias_mu || !L.bias_sigma || !L.noise_in ||
        !L.noise_out || !L.weight || !L.bias)
      return false;
  }
  return true;
}

unsigned blocks_for(long long n) {
  const long long b = (n + kThreads - 1) / kThreads;
  return (unsigned)(b < 1 ? 1 : b > kMaxBlocks ? kMaxBlocks : b);
}

}  // namespace

WDB_API int wdb_noisy_supported(const wdb_noisy_net *net) { return shape_ok(net); }

WDB_API int wdb_noisy_draw(void *stream, const wdb_noisy_net *net, unsigned long long seed,
                           int domain, unsigned long long count, int row0, int n_rows) {
  if (!shape_ok(net) || n_rows < 1 || row0 < 0 || (domain != 0 && domain != 1))
    return (int)cudaErrorInvalidValue;
  for (int l = 0; l < net->n_layers; ++l)
    if (!net->layer[l].noise_in || !net->layer[l].noise_out) return (int)cudaErrorInvalidValue;
  long long per_row = 0;
  for (int l = 0; l < net->n_layers; ++l) per_row += net->layer[l].in_dim + net->layer[l].out_dim;
  noisy_draw_kernel<<<blocks_for(per_row * n_rows), kThreads, 0, as_stream(stream)>>>(
      *net, seed, domain, count, row0, n_rows);
  return finish_launch();
}

WDB_API int wdb_noisy_materialize(void *stream, const wdb_noisy_net *online,
                                  const wdb_noisy_net *target, unsigned long long seed,
                                  unsigned long long update) {
  if (!shape_ok(online) || !materialize_pointers_ok(*online)) return (int)cudaErrorInvalidValue;
  if (target && (!same_shape(*online, *target) || !materialize_pointers_ok(*target)))
    return (int)cudaErrorInvalidValue;
  const dim3 grid(blocks_for(total(*online, true)), target ? 2 : 1);
  noisy_materialize_kernel<<<grid, kThreads, 0, as_stream(stream)>>>(
      *online, target ? *target : *online, seed, update);
  return finish_launch();
}

WDB_API int wdb_noisy_grads(void *stream, const wdb_noisy_net *net) {
  if (!shape_ok(net)) return (int)cudaErrorInvalidValue;
  for (int l = 0; l < net->n_layers; ++l) {
    const wdb_noisy_layer &L = net->layer[l];
    if (!L.noise_in || !L.noise_out || !L.grad_weight || !L.grad_bias || !L.grad_weight_mu ||
        !L.grad_weight_sigma || !L.grad_bias_mu || !L.grad_bias_sigma)
      return (int)cudaErrorInvalidValue;
  }
  noisy_grads_kernel<<<blocks_for(total(*net, false)), kThreads, 0, as_stream(stream)>>>(*net);
  return finish_launch();
}
