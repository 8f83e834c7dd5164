// The listwise AP loss of "Learning with Average Precision" (reference dirtorch/loss.py), forward and backward, without
// the N x 2nq x M tensor the reference's 1x1 Conv1d quantiser materialises (dirb200_aploss_forward / _backward).
//
// Quantiser (loss.py:29-41): 2nq lines v_i = w_i x + b_i, bin j = max(0, min(v_j, v_{j+nq})), evaluated here as
// fl32(fmaf(w_i, x, b_i)).  With p = v_1 = fmaf(w_1, x, b_1), bin j peaks at p = j and is non-zero on |p - j| < 1, so
// every bin whose pre-clamp value is >= 0 (the bins that receive a gradient under torch's clamp convention) lies in
// {k - 1, k, k + 1}, k = rint(p): p is within a few ulps of its exact value, far less than the 1/2 this needs.  Those
// three candidates are evaluated with the exact table formula; every decision (clamp, min branch, tie) is taken on
// the fp32 v values, as the reference takes it.
//
//   1. aploss_hist_kernel: per row n and bin j, c = sum_m q_j(x_nm) and cp = sum_m q_j(x_nm) l_nm, and the positive
//      count, in fixed point (q rounded to nearest in units of 2^-32, int64).  Integer sums are exact and order-free:
//      the histogram does not depend on the grid, on the schedule or on the other rows of the call.  A thread keeps
//      the three bins around its first element's k in registers (concentrated scores land there); other elements are
//      aggregated across the warp by __match_any_sync, one shared int64 atomic per distinct bin, and each CTA adds its
//      shared histogram to the caller's with global int64 atomics.  No float atomics.
//   2. aploss_final_kernel: one warp per row, fp64.  AP (or TAP) of the row and the gradient coefficients
//      G = [dAP/dc | dAP/dcp], computed by lane 0 in bin order (the order tests/aploss_model.py uses).
//   3. aploss_backward_kernel: dx = fl32(grad_ap * sum_{active j} (G_c[j] + l G_cp[j]) q_j'(x)), with q_j' = w of the
//      smaller branch of the min, the mean of both on a tie; bins whose min is < 0 are left out.  An active bin with a
//      zero slope (x beyond the range, or at a bin's peak) still multiplies its coefficient, so a row whose G is NaN
//      (no positive) gets NaN everywhere, as the reference's conv backward gives it.
#include <limits.h>
#include <math.h>

#include "common.h"

namespace dirb {
namespace {

constexpr int AP_THREADS = 256;
constexpr int64_t AP_CHUNK = AP_THREADS * 64;   // elements of one row per work item
constexpr int AP_MAX_NQ = 100;
constexpr float FIX_SCALE = 4294967296.0f;      // 2^32
constexpr int FIN_WARPS = 4;

struct Quant {
  const float2* bias;   // shared: (b_j, b_{j+nq})
  float w1, w0, wn, wl;  // w_1 (= w_j, 1 <= j < nq), w_0, w_nq (= w_{j+nq}, j < nq - 1), w_{2nq-1}
  int nq;

  __device__ __forceinline__ int center(float x) const {
    const float p = fmaf(w1, x, bias[1].x);
    return __float2int_rn(fminf(fmaxf(p, -1.0f), static_cast<float>(nq)));   // NaN -> -1
  }
  // pre-clamp value min(v_j, v_{j+nq}) and the slope of the branch the min takes (the mean of both on a tie)
  __device__ __forceinline__ float eval(int j, float x, float& slope) const {
    const float2 b = bias[j];
    const float wlo = j == 0 ? w0 : w1, whi = j == nq - 1 ? wl : wn;
    const float vlo = fmaf(wlo, x, b.x), vhi = fmaf(whi, x, b.y);
    slope = vlo < vhi ? wlo : (vlo > vhi ? whi : 0.5f * (wlo + whi));   // exact: wlo + whi is 0 or +-a
    return fminf(vlo, vhi);
  }
};

__device__ __forceinline__ void load_quant(Quant& q, const float* __restrict__ table, int nq, float2* bias_s) {
  for (int j = threadIdx.x; j < nq; j += blockDim.x) bias_s[j] = make_float2(table[2 * nq + j], table[3 * nq + j]);
  q.bias = bias_s;
  q.w1 = table[1];
  q.w0 = table[0];
  q.wn = table[nq];
  q.wl = table[2 * nq - 1];
  q.nq = nq;
}

__device__ __forceinline__ long long fixq(float v) {
  return v > 0.0f ? __float2ll_rn(v * FIX_SCALE) : 0ll;   // v * 2^32 is exact
}

// grid-stride over (row, chunk) items.  hist[n][0, nq) = c, [nq, 2nq) = cp, [2nq] = positives, units 2^-32.
__global__ void __launch_bounds__(AP_THREADS) aploss_hist_kernel(const float* __restrict__ x,
                                                                 const uint8_t* __restrict__ label, int64_t N,
                                                                 int64_t M, int nq, const float* __restrict__ table,
                                                                 unsigned long long* __restrict__ hist) {
  __shared__ float2 bias_s[AP_MAX_NQ];
  __shared__ unsigned long long h_s[2 * AP_MAX_NQ + 1];
  __shared__ long long stage[AP_THREADS / 32][32][4];
  Quant q;
  load_quant(q, table, nq, bias_s);
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int H = 2 * nq + 1;
  const int64_t chunks = (M + AP_CHUNK - 1) / AP_CHUNK;
  const int64_t items = N * chunks;
  for (int64_t it = blockIdx.x; it < items; it += gridDim.x) {
    const int64_t n = it / chunks, m0 = (it % chunks) * AP_CHUNK;
    const int64_t m1 = min(M, m0 + AP_CHUNK);
    for (int j = tid; j < H; j += AP_THREADS) h_s[j] = 0ull;
    __syncthreads();
    const float* xr = x + n * M;
    const uint8_t* lr = label + n * M;
    long long acc_c[3] = {0, 0, 0}, acc_p[3] = {0, 0, 0};
    int key = INT_MIN, npos = 0;
    for (int64_t base = m0; base < m1; base += AP_THREADS * 8) {
      float xv[8];
      uint8_t lv[8];
#pragma unroll
      for (int u = 0; u < 8; ++u) {
        const int64_t m = base + u * AP_THREADS + tid;
        xv[u] = m < m1 ? __ldg(xr + m) : 0.0f;
        lv[u] = m < m1 ? __ldg(lr + m) : 0;
      }
#pragma unroll
      for (int u = 0; u < 8; ++u) {
        const bool valid = base + u * AP_THREADS + tid < m1;
        const int k = q.center(xv[u]);
        const bool pos = valid && lv[u] != 0;
        long long f[3];
#pragma unroll
        for (int s = 0; s < 3; ++s) {
          const int j = k - 1 + s;
          float slope;
          f[s] = (j >= 0 && j < nq) ? fixq(q.eval(j, xv[u], slope)) : 0ll;
        }
        npos += pos;
        if (valid && key == INT_MIN) key = k;
        const bool hit = valid && k == key;
        if (hit) {
#pragma unroll
          for (int s = 0; s < 3; ++s) {
            acc_c[s] += f[s];
            acc_p[s] += pos ? f[s] : 0ll;
          }
        }
        const bool miss = valid && !hit;
        if (__any_sync(0xffffffffu, miss)) {
          const unsigned peers = __match_any_sync(0xffffffffu, miss ? k : INT_MIN);
          if (miss) {
            stage[warp][lane][0] = f[0];
            stage[warp][lane][1] = f[1];
            stage[warp][lane][2] = f[2];
            stage[warp][lane][3] = pos;
          }
          __syncwarp();
          if (miss && lane == __ffs(peers) - 1) {
            long long sc[3] = {0, 0, 0}, sp[3] = {0, 0, 0};
            for (unsigned r = peers; r; r &= r - 1) {
              const long long* e = stage[warp][__ffs(r) - 1];
#pragma unroll
              for (int s = 0; s < 3; ++s) {
                sc[s] += e[s];
                sp[s] += e[3] ? e[s] : 0ll;
              }
            }
#pragma unroll
            for (int s = 0; s < 3; ++s) {
              const int j = k - 1 + s;
              if (sc[s]) atomicAdd(&h_s[j], static_cast<unsigned long long>(sc[s]));
              if (sp[s]) atomicAdd(&h_s[nq + j], static_cast<unsigned long long>(sp[s]));
            }
          }
          __syncwarp();
        }
      }
    }
    // flush the register bins: one warp reduction when the whole warp shares its key, else one atomic per thread
    const int key0 = __shfl_sync(0xffffffffu, key, 0);
    if (__all_sync(0xffffffffu, key == key0 || key == INT_MIN)) {
#pragma unroll
      for (int s = 0; s < 3; ++s)
#pragma unroll
        for (int o = 16; o; o >>= 1) {
          acc_c[s] += __shfl_xor_sync(0xffffffffu, acc_c[s], o);
          acc_p[s] += __shfl_xor_sync(0xffffffffu, acc_p[s], o);
        }
      if (lane != 0) key = INT_MIN;
      else key = key0;
    }
    if (key != INT_MIN) {
#pragma unroll
      for (int s = 0; s < 3; ++s) {
        const int j = key - 1 + s;
        if (acc_c[s]) atomicAdd(&h_s[j], static_cast<unsigned long long>(acc_c[s]));
        if (acc_p[s]) atomicAdd(&h_s[nq + j], static_cast<unsigned long long>(acc_p[s]));
      }
    }
    const unsigned pw = __reduce_add_sync(0xffffffffu, static_cast<unsigned>(npos));
    if (lane == 0 && pw) atomicAdd(&h_s[2 * nq], static_cast<unsigned long long>(pw) << 32);
    __syncthreads();
    for (int j = tid; j < H; j += AP_THREADS)
      if (h_s[j]) atomicAdd(hist + n * H + j, h_s[j]);
    __syncthreads();   // h_s is reset by the next item
  }
}

// one warp per row; the warp moves the row in and out, lane 0 runs the recurrences in bin order.
// mode 0: APLoss (loss.py:50-55), eps 1e-16.  mode 1 / 2: TAPLoss (loss.py:97-119), full / simplified, eps 1e-8.
__global__ void __launch_bounds__(FIN_WARPS * 32) aploss_final_kernel(const unsigned long long* __restrict__ hist,
                                                                      int64_t N, int nq, int mode,
                                                                      double* __restrict__ G, float* __restrict__ ap) {
  __shared__ double s_c[FIN_WARPS][AP_MAX_NQ], s_p[FIN_WARPS][AP_MAX_NQ];
  __shared__ double s_C[FIN_WARPS][AP_MAX_NQ], s_P[FIN_WARPS][AP_MAX_NQ];
  __shared__ double s_g[FIN_WARPS][2 * AP_MAX_NQ], s_L[FIN_WARPS][AP_MAX_NQ];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int64_t n = static_cast<int64_t>(blockIdx.x) * FIN_WARPS + warp;
  if (n >= N) return;
  const int H = 2 * nq + 1;
  const double unit = 1.0 / 4294967296.0;
  double* c = s_c[warp];
  double* cp = s_p[warp];
  double* C = s_C[warp];
  double* P = s_P[warp];
  double* g = s_g[warp];
  double* Ls = s_L[warp];
  for (int j = lane; j < nq; j += 32) {
    c[j] = static_cast<double>(static_cast<long long>(hist[n * H + j])) * unit;
    cp[j] = static_cast<double>(static_cast<long long>(hist[n * H + nq + j])) * unit;
  }
  __syncwarp();
  if (lane == 0) {
    double sc = 0.0, sp = 0.0;
    for (int j = 0; j < nq; ++j) {
      sc += c[j];
      sp += cp[j];
      C[j] = sc;
      P[j] = sp;
    }
  }
  __syncwarp();
  // TAP's logs, one bin per lane (kept out of lane 0's recurrences, which then need no call)
  if (mode == 1)
    for (int j = lane; j < nq; j += 32) Ls[j] = log((C[j] + 1.0) / ((j ? C[j - 1] : 0.0) + 1.0));
  __syncwarp();
  if (lane == 0) {
    double res = 0.0;
    if (mode == 0) {
      const double eps = 1e-16, S = P[nq - 1];
      for (int j = 0; j < nq; ++j) res += (P[j] / (eps + C[j])) * (cp[j] / S);
      double a1 = 0.0, a2 = 0.0;
      for (int k = nq - 1; k >= 0; --k) {
        const double d = eps + C[k], A = P[k] / d, u = cp[k] / S;
        a1 += u * A / d;
        a2 += u / d;
        g[k] = -a1;
        g[nq + k] = A / S + a2 - res / S;
      }
    } else {
      const double Np = static_cast<double>(static_cast<long long>(hist[n * H + 2 * nq])) * unit;
      if (mode == 2) {
        for (int j = 0; j < nq; ++j) {
          const double C1 = j ? C[j - 1] : 0.0, P1 = j ? P[j - 1] : 0.0;
          res += cp[j] * (P1 + P[j] + 1.0) / (C1 + C[j] + 1.0) / Np;
        }
        double sa = 0.0, sb = 0.0;   // sum_{j>k} ap_j / D_j, sum_{j>k} cp_j / (D_j Np)
        for (int k = nq - 1; k >= 0; --k) {
          const double C1 = k ? C[k - 1] : 0.0, P1 = k ? P[k - 1] : 0.0;
          const double D = C1 + C[k] + 1.0, Nu = P1 + P[k] + 1.0;
          const double apk = cp[k] * Nu / D / Np;
          g[k] = -apk / D - 2.0 * sa;
          g[nq + k] = (Nu + cp[k]) / (D * Np) + 2.0 * sb;
          sa += apk / D;
          sb += cp[k] / (D * Np);
        }
      } else {
        const double eps = 1e-8;
        // ap_j = E_j T_j with E_j = cp_j / (c_j + eps) / Np, T_j = c_j r_j + B_j L_j, B_j = P_{j-1} + 1 - r_j (C_{j-1} + 1),
        // L_j = log((C_j + 1) / (C_{j-1} + 1)), r_j = relu(cp_j - 1) / (relu(c_j - 1) + eps).  c_k reaches C_j (j >= k,
        // coefficient alpha_j) and C_{j-1} (j > k, beta_j); cp_k reaches P_{j-1} (j > k, gamma_j = E_j L_j).
        double sab = 0.0, sg = 0.0;   // sum_{j>=k} alpha_j + sum_{j>k} beta_j ; sum_{j>k} gamma_j
        double beta_next = 0.0;
        for (int k = nq - 1; k >= 0; --k) {
          const double C1 = k ? C[k - 1] : 0.0, P1 = k ? P[k - 1] : 0.0;
          const double hc = c[k] - 1.0, hp = cp[k] - 1.0;
          const double den = fmax(hc, 0.0) + eps;
          const double r = fmax(hp, 0.0) / den;
          const double L = Ls[k];
          const double B = P1 + 1.0 - r * (C1 + 1.0);
          const double T = c[k] * r + B * L;
          const double E = cp[k] / (c[k] + eps) / Np;
          const double apk = cp[k] * T / (c[k] + eps) / Np;
          const double alpha = E * B / (C[k] + 1.0);
          const double beta = E * (-r * L - B / (C1 + 1.0));
          const double rho = E * (c[k] - (C1 + 1.0) * L);
          sab += alpha + beta_next;
          beta_next = beta;
          const double dr_dc = hc >= 0.0 ? -r / den : 0.0, dr_dp = hp >= 0.0 ? 1.0 / den : 0.0;
          g[k] = -apk / (c[k] + eps) + E * r + rho * dr_dc + sab;
          g[nq + k] = T / ((c[k] + eps) * Np) + rho * dr_dp + sg;
          sg += E * L;
        }
        // the loss sums in bin order, as the reference
        for (int j = 0; j < nq; ++j) {
          const double C1 = j ? C[j - 1] : 0.0, P1 = j ? P[j - 1] : 0.0;
          const double r = fmax(cp[j] - 1.0, 0.0) / (fmax(c[j] - 1.0, 0.0) + eps);
          const double L = Ls[j];
          res += cp[j] * (c[j] * r + (P1 + 1.0 - r * (C1 + 1.0)) * L) / (c[j] + eps) / Np;
        }
      }
    }
    ap[n] = static_cast<float>(res);
  }
  __syncwarp();
  for (int j = lane; j < 2 * nq; j += 32) G[n * 2 * nq + j] = g[j];
}

__global__ void __launch_bounds__(AP_THREADS) aploss_backward_kernel(const float* __restrict__ x,
                                                                     const uint8_t* __restrict__ label, int64_t N,
                                                                     int64_t M, int nq, const float* __restrict__ table,
                                                                     const double* __restrict__ G,
                                                                     const float* __restrict__ grad_ap,
                                                                     float* __restrict__ dx) {
  __shared__ float2 bias_s[AP_MAX_NQ];
  __shared__ double2 g_s[AP_MAX_NQ];   // (dAP/dc_j, dAP/dcp_j)
  Quant q;
  load_quant(q, table, nq, bias_s);
  const int tid = threadIdx.x;
  const int64_t chunks = (M + AP_CHUNK - 1) / AP_CHUNK;
  const int64_t items = N * chunks;
  int64_t row = -1;
  for (int64_t it = blockIdx.x; it < items; it += gridDim.x) {
    const int64_t n = it / chunks, m0 = (it % chunks) * AP_CHUNK;
    const int64_t m1 = min(M, m0 + AP_CHUNK);
    if (n != row) {
      __syncthreads();
      for (int j = tid; j < nq; j += AP_THREADS) g_s[j] = make_double2(G[n * 2 * nq + j], G[n * 2 * nq + nq + j]);
      row = n;
    }
    __syncthreads();
    const double ga = static_cast<double>(grad_ap[n]);
    const float* xr = x + n * M;
    const uint8_t* lr = label + n * M;
    float* dr = dx + n * M;
    for (int64_t base = m0; base < m1; base += AP_THREADS * 8) {
      float xv[8];
      uint8_t lv[8];
#pragma unroll
      for (int u = 0; u < 8; ++u) {
        const int64_t m = base + u * AP_THREADS + tid;
        xv[u] = m < m1 ? __ldg(xr + m) : 0.0f;
        lv[u] = m < m1 ? __ldg(lr + m) : 0;
      }
#pragma unroll
      for (int u = 0; u < 8; ++u) {
        const int64_t m = base + u * AP_THREADS + tid;
        const int k = q.center(xv[u]);
        double s = 0.0;
#pragma unroll
        for (int t = 0; t < 3; ++t) {
          const int j = k - 1 + t;
          if (j >= 0 && j < nq) {
            float slope;
            if (q.eval(j, xv[u], slope) >= 0.0f) {   // a zero slope still carries a NaN G, as in torch
              const double2 gj = g_s[j];
              s += (lv[u] ? gj.x + gj.y : gj.x) * static_cast<double>(slope);
            }
          }
        }
        if (m < m1) dr[m] = static_cast<float>(ga * s);
      }
    }
  }
}

int check_args(const float* x, const uint8_t* label, int64_t N, int64_t M, int nq, const float* table,
               const char* who) {
  DIRB_REQUIRE(N >= 1 && M >= 1, DIRB200_EINVAL, "%s: bad shape N %lld, M %lld", who, (long long)N, (long long)M);
  DIRB_REQUIRE(nq >= 2 && nq <= AP_MAX_NQ, DIRB200_EINVAL, "%s: nq %d outside [2, %d]", who, nq, AP_MAX_NQ);
  DIRB_REQUIRE(x && label && table, DIRB200_EINVAL, "%s: null argument", who);
  DIRB_REQUIRE(M < (int64_t(1) << 31), DIRB200_ENOTSUP,
               "%s: M %lld >= 2^31 (the int64 fixed-point histogram could overflow)", who, (long long)M);
  return require_sm90();
}

unsigned grid_for(int64_t N, int64_t M) {
  const int64_t items = N * ceil_div(M, AP_CHUNK);
  return static_cast<unsigned>(items < 0x7fffffff ? items : 0x7fffffff);
}

}  // namespace
}  // namespace dirb

using namespace dirb;

extern "C" {

int dirb200_aploss_forward(const float* x_dev, const uint8_t* label_dev, int64_t N, int64_t M, int nq,
                           const float* table_dev, int mode, int64_t* hist_dev, double* G_dev, float* ap_dev,
                           void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  DIRB_TRY(check_args(x_dev, label_dev, N, M, nq, table_dev, "aploss_forward"));
  DIRB_REQUIRE(mode >= 0 && mode <= 2, DIRB200_EINVAL, "aploss_forward: mode %d not in {0, 1, 2}", mode);
  DIRB_REQUIRE(hist_dev && G_dev && ap_dev, DIRB200_EINVAL, "aploss_forward: null output");
  DIRB_CUDA(cudaMemsetAsync(hist_dev, 0, static_cast<size_t>(N) * (2 * nq + 1) * 8, stream));
  aploss_hist_kernel<<<grid_for(N, M), AP_THREADS, 0, stream>>>(x_dev, label_dev, N, M, nq, table_dev,
                                                                reinterpret_cast<unsigned long long*>(hist_dev));
  aploss_final_kernel<<<static_cast<unsigned>(ceil_div(N, FIN_WARPS)), FIN_WARPS * 32, 0, stream>>>(
      reinterpret_cast<const unsigned long long*>(hist_dev), N, nq, mode, G_dev, ap_dev);
  count_launch(2);
  DIRB_CUDA(cudaGetLastError());
  return 0;
}

int dirb200_aploss_backward(const float* x_dev, const uint8_t* label_dev, int64_t N, int64_t M, int nq,
                            const float* table_dev, const double* G_dev, const float* grad_ap_dev, float* dx_dev,
                            void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  DIRB_TRY(check_args(x_dev, label_dev, N, M, nq, table_dev, "aploss_backward"));
  DIRB_REQUIRE(G_dev && grad_ap_dev && dx_dev, DIRB200_EINVAL, "aploss_backward: null argument");
  aploss_backward_kernel<<<grid_for(N, M), AP_THREADS, 0, stream>>>(x_dev, label_dev, N, M, nq, table_dev, G_dev,
                                                                    grad_ap_dev, dx_dev);
  count_launch(1);
  DIRB_CUDA(cudaGetLastError());
  return 0;
}

}  // extern "C"
