// loaders.cuh -- operand loaders and epilogues that turn every dense contraction of the IMPALA
// actor-critic (model/impala_actor_critic.py:5-42) and its backward pass into the gather-GEMM of
// gemm_simt.cuh.  Activations are NHWC float32 with TIME-MAJOR rows (row m = t*B + b) so that
// the B*(T-2) rows that receive gradient (optimizer/vtrace.py:10, agent/impala.py:78-93) are the
// contiguous prefix; the fed inputs (frames, h, c, prev_action) stay in the caller's batch-major
// [B,T,...] layout and are addressed through the (t,b) -> b*T+t remap.
#pragma once
#include "common.cuh"
#include "split16.cuh"

namespace drl {

__device__ __forceinline__ float4 u8x4_to_f4(uchar4 u) {
  return make_float4((float)u.x, (float)u.y, (float)u.z, (float)u.w);
}
// 4 bytes -> 4 floats without the XU-pipe I2F: PRMT builds the bit pattern of 2^23 + b (0x4B0000bb), one FADD removes
// the 2^23 (exact for b in [0, 255]).  ncu showed the XU pipe ~29 % busy with I2F.U8 in the conv1 kernels.
__device__ __forceinline__ float4 u32_bytes_to_f4(uint32_t w) {
  const float m = 8388608.0f;
  return make_float4(__uint_as_float(__byte_perm(w, 0x4B000000u, 0x7650)) - m,
                     __uint_as_float(__byte_perm(w, 0x4B000000u, 0x7651)) - m,
                     __uint_as_float(__byte_perm(w, 0x4B000000u, 0x7652)) - m,
                     __uint_as_float(__byte_perm(w, 0x4B000000u, 0x7653)) - m);
}
// 16 frame bytes (one 128-bit load) -> 16 floats
__device__ __forceinline__ void unpack_u8x16(const uint4& u, float4 (&f)[4]) {
  f[0] = u32_bytes_to_f4(u.x); f[1] = u32_bytes_to_f4(u.y); f[2] = u32_bytes_to_f4(u.z); f[3] = u32_bytes_to_f4(u.w);
}

// time-major row index -> batch-major source index
struct RowMap {
  int B, T;
  __device__ __forceinline__ int src(int m) const {
    const int t = m / B;
    const int b = m - t * B;
    return b * T + t;
  }
};

// --------------------------------------------------------------------------------------------
// Forward convolution A operand (im2col gather), K-contiguous: k = (ky*KW + kx)*C + ci.
// For NHWC input a fixed ky gives a run of KW*C contiguous elements.
// --------------------------------------------------------------------------------------------
template <typename T, int IH, int IW, int C, int OH, int OW, int KW, int S, bool REMAP>
struct ConvFwdA {
  static constexpr bool kContigK = true;
  static constexpr bool kExactTf32 = (sizeof(T) == 1);   // uint8 frame bytes are exact in tf32
  const T* x;
  RowMap map;
  struct Row { const T* base; };
  __device__ __forceinline__ Row row(int, int m) const {
    Row r;
    if (m < 0) { r.base = nullptr; return r; }
    const int img = m / (OH * OW);
    const int p = m - img * (OH * OW);
    const int oy = p / OW, ox = p - oy * OW;
    const int simg = REMAP ? map.src(img) : img;
    r.base = x + (size_t)simg * (IH * IW * C) + ((oy * S) * IW + ox * S) * C;
    return r;
  }
  // address of element k of row r (nullptr: the row is out of range); a run of KW*C elements along k is contiguous
  __device__ __forceinline__ const T* addr(const Row& r, int k) const {
    if (r.base == nullptr) return nullptr;
    const int ky = k / (KW * C);
    const int rr = k - ky * (KW * C);
    return r.base + ky * (IW * C) + rr;
  }
  __device__ __forceinline__ float4 load(const Row& r, int k) const {
    const T* p = addr(r, k);
    if (p == nullptr) return zero4();
    if constexpr (sizeof(T) == 1) {
      return u8x4_to_f4(__ldg(reinterpret_cast<const uchar4*>(p)));
    } else {
      return __ldg(reinterpret_cast<const float4*>(p));
    }
  }
  // uint8 operands: 16 consecutive k (k multiple of 16) are 16 contiguous, 16-byte aligned frame bytes
  static constexpr bool kVec16 = (sizeof(T) == 1) && ((KW * C) % 16 == 0);
  __device__ __forceinline__ uint4 load_raw16(const Row& r, int k) const {
    if (r.base == nullptr) return make_uint4(0u, 0u, 0u, 0u);
    const int ky = k / (KW * C);
    const int rr = k - ky * (KW * C);
    return __ldg(reinterpret_cast<const uint4*>(r.base + ky * (IW * C) + rr));
  }
  __device__ static __forceinline__ void unpack16(const uint4& u, float4 (&f)[4]) { unpack_u8x16(u, f); }
};

// Weight-gradient A operand: C[i, co] = sum_r X(i, r) dY(r, co); i = (ky,kx,ci) is the contiguous
// ("M-major") index, r = (img, oy, ox) the reduction index.
template <typename T, int IH, int IW, int C, int OH, int OW, int KW, int S, bool REMAP>
struct ConvWgradA {
  static constexpr bool kContigK = false;
  static constexpr bool kExactTf32 = (sizeof(T) == 1);
  const T* x;
  RowMap map;
  struct Row { int off; };
  __device__ __forceinline__ Row row(int, int i) const {
    Row r;
    if (i < 0) { r.off = -1; return r; }
    const int ky = i / (KW * C);
    r.off = ky * (IW * C) + (i - ky * (KW * C));
    return r;
  }
  __device__ __forceinline__ float4 load(const Row& r, int rr) const {
    if (r.off < 0) return zero4();
    const int img = rr / (OH * OW);
    const int p = rr - img * (OH * OW);
    const int oy = p / OW, ox = p - oy * OW;
    const int simg = REMAP ? map.src(img) : img;
    const T* ptr = x + (size_t)simg * (IH * IW * C) + ((oy * S) * IW + ox * S) * C + r.off;
    if constexpr (sizeof(T) == 1) {
      return u8x4_to_f4(__ldg(reinterpret_cast<const uchar4*>(ptr)));
    } else {
      return __ldg(reinterpret_cast<const float4*>(ptr));
    }
  }
  // uint8 operands: 16 consecutive features i (i multiple of 16) of one output pixel are 16 contiguous bytes
  static constexpr bool kVec16 = (sizeof(T) == 1) && ((KW * C) % 16 == 0) && ((S * C) % 16 == 0);
  __device__ __forceinline__ uint4 load_raw16(const Row& r, int rr) const {
    if (r.off < 0) return make_uint4(0u, 0u, 0u, 0u);
    const int img = rr / (OH * OW);
    const int p = rr - img * (OH * OW);
    const int oy = p / OW, ox = p - oy * OW;
    const int simg = REMAP ? map.src(img) : img;
    return __ldg(reinterpret_cast<const uint4*>(x + (size_t)simg * (IH * IW * C) + ((oy * S) * IW + ox * S) * C + r.off));
  }
  __device__ static __forceinline__ void unpack16(const uint4& u, float4 (&f)[4]) { unpack_u8x16(u, f); }
};

// Data-gradient A operand (gather form): rows are input pixels of parity class z = (py,px)
// (S*S classes; one class when S = 1), k = (tap, co) with tap = (jy, jx), ky = py + S*jy.
//   dX[img, yy*S+py, xx*S+px, ci] = sum_{jy,jx,co} dY[img, yy-jy, xx-jx, co] * W[ky,kx,ci,co]
template <int OH, int OW, int CO, int S, int KH, int KW, int RH, int RW>
struct ConvDgradA {
  static constexpr bool kContigK = true;
  static constexpr int TW = KW / S;
  const float* dy;
  struct Row { int img, yy, xx; };
  __device__ __forceinline__ Row row(int, int m) const {
    Row r;
    if (m < 0) { r.img = -1; r.yy = 0; r.xx = 0; return r; }
    r.img = m / (RH * RW);
    const int p = m - r.img * (RH * RW);
    r.yy = p / RW;
    r.xx = p - r.yy * RW;
    return r;
  }
  // address of element k of row r (nullptr: row out of range or tap outside the output: zero); CO elements per tap
  __device__ __forceinline__ const float* addr(const Row& r, int k) const {
    if (r.img < 0) return nullptr;
    const int tap = k / CO;
    const int co = k - tap * CO;
    const int jy = tap / TW, jx = tap - jy * TW;
    const int oy = r.yy - jy, ox = r.xx - jx;
    if (oy < 0 || oy >= OH || ox < 0 || ox >= OW) return nullptr;
    return dy + ((size_t)(r.img * OH + oy) * OW + ox) * CO + co;
  }
  __device__ __forceinline__ float4 load(const Row& r, int k) const {
    const float* p = addr(r, k);
    return p ? __ldg(reinterpret_cast<const float4*>(p)) : zero4();
  }
};
// Matching B operand: B(k=(tap,co), n=ci) = W[ky, kx, ci, co], contiguous along co (= along k).
template <int CI, int CO, int S, int KH, int KW>
struct ConvDgradB {
  static constexpr bool kContigK = true;
  static constexpr int TW = KW / S;
  const float* w;   // HWIO
  struct Row { int n, py, px; };
  __device__ __forceinline__ Row row(int z, int n) const {
    Row r;
    r.n = n;
    r.py = z / S;
    r.px = z - r.py * S;
    return r;
  }
  __device__ __forceinline__ float4 load(const Row& r, int k) const {
    if (r.n < 0) return zero4();
    const int tap = k / CO;
    const int co = k - tap * CO;
    const int jy = tap / TW, jx = tap - jy * TW;
    const int ky = r.py + S * jy, kx = r.px + S * jx;
    return __ldg(reinterpret_cast<const float4*>(w + ((size_t)((ky * KW + kx) * CI + r.n)) * CO + co));
  }
};
// All S*S parity classes side by side along N: n = (z, ci), B(k, n) = class z's B(k, ci).  Every class of the S x S block
// of input pixels at (yy, xx) reads the same dY taps, so the whole data gradient is ONE GEMM with N = S*S*CI whose A
// operand (ConvDgradA) is gathered once per row instead of once per class.
template <int CI, int CO, int S, int KH, int KW>
struct ConvDgradBMerged {
  static constexpr bool kContigK = true;
  ConvDgradB<CI, CO, S, KH, KW> b;
  using Row = typename ConvDgradB<CI, CO, S, KH, KW>::Row;
  __device__ __forceinline__ Row row(int, int n) const { return n < 0 ? b.row(0, -1) : b.row(n / CI, n % CI); }
  __device__ __forceinline__ float4 load(const Row& r, int k) const { return b.load(r, k); }
};

// A K-major A operand read from the 16-bit plane (Plane16) of the fp32 buffer `base` that loader L gathers from: the same
// rows and the same gather addresses as L, as element indices into the plane.  gemm_umma16_kernel copies each 16-byte
// chunk (8 consecutive k: L's contiguous runs along k are multiples of 8 long) of hi and of lo straight into the stage
// with cp.async: no operand registers, no conversion, and the bits of the fp32 path.
template <class L>
struct PlaneA {
  static_assert(L::kContigK, "plane operands are K-major");
  static constexpr bool kContigK = true;
  static constexpr bool kPlane = true;
  L l;
  const float* base;        // the fp32 buffer L reads
  const uint16_t* plane;    // its [hi | lo] plane
  size_t count;             // elements of the buffer (offset of the lo half)
  using Row = typename L::Row;
  __device__ __forceinline__ Row row(int z, int m) const { return l.row(z, m); }
  // element index of the chunk [k, k + 8) of row r (k a multiple of 8), or -1: zero
  __device__ __forceinline__ long long chunk(const Row& r, int k) const {
    const float* p = l.addr(r, k);
    return p ? (long long)(p - base) : -1ll;
  }
};

// --------------------------------------------------------------------------------------------
// LSTM operand: x_m = [flatten(a3_m) | emb[prev_action_m] | h0_m]  (model/impala_actor_critic.py:35-38,
// TF LSTMCell concat order: inputs then h).
// --------------------------------------------------------------------------------------------
struct LstmA {   // K-contiguous rows
  static constexpr bool kContigK = true;
  const float* e;       // [M, 3136] time-major
  const float* table;   // [A, 256]
  const int* pa;        // [B, T] batch-major
  const float* h0;      // [B, T, 256] batch-major
  RowMap map;
  struct Row { const float *pe, *pu, *ph; };
  __device__ __forceinline__ Row row(int, int m) const {
    Row r;
    if (m < 0) { r.pe = nullptr; r.pu = nullptr; r.ph = nullptr; return r; }
    const int s = map.src(m);
    r.pe = e + (size_t)m * Geo::FLAT;
    r.pu = table + (size_t)__ldg(pa + s) * Geo::EMB - Geo::FLAT;
    r.ph = h0 + (size_t)s * Geo::L - (Geo::FLAT + Geo::EMB);
    return r;
  }
  __device__ __forceinline__ float4 load(const Row& r, int k) const {
    if (r.pe == nullptr) return zero4();
    const float* p = (k < Geo::FLAT) ? r.pe : ((k < Geo::FLAT + Geo::EMB) ? r.pu : r.ph);
    return __ldg(reinterpret_cast<const float4*>(p + k));
  }
};
struct LstmAT {  // transposed view for dW = X^T dz : index i = feature (contiguous), reduction r = row
  static constexpr bool kContigK = false;
  const float* e;
  const float* table;
  const int* pa;
  const float* h0;
  RowMap map;
  struct Row { int i; };
  __device__ __forceinline__ Row row(int, int i) const { Row r; r.i = i; return r; }
  __device__ __forceinline__ float4 load(const Row& r, int m) const {
    if (r.i < 0) return zero4();
    const float* p;
    if (r.i < Geo::FLAT) {
      p = e + (size_t)m * Geo::FLAT + r.i;
    } else {
      const int s = map.src(m);
      if (r.i < Geo::FLAT + Geo::EMB) p = table + (size_t)__ldg(pa + s) * Geo::EMB + (r.i - Geo::FLAT);
      else p = h0 + (size_t)s * Geo::L + (r.i - Geo::FLAT - Geo::EMB);
    }
    return __ldg(reinterpret_cast<const float4*>(p));
  }
};
// [x | h_in]^T for the LSTM kernel gradient of an unrolled LSTM (the R2D2 learner; the IMPALA learner's recurrent mode):
// feature index i < 3392 -> [a3 | emb] (as LstmAT), else h_in, the state the recurrence read (device, time-major [M, L])
struct LstmHinAT {
  static constexpr bool kContigK = false;
  const float* e; const float* table; const int* pa; const float* hin; RowMap map; int L;
  struct Row { int i; };
  __device__ __forceinline__ Row row(int, int i) const { Row r; r.i = i; return r; }
  __device__ __forceinline__ float4 load(const Row& r, int m) const {
    if (r.i < 0) return zero4();
    const float* p;
    if (r.i < Geo::FLAT) p = e + (size_t)m * Geo::FLAT + r.i;
    else if (r.i < Geo::FLAT + Geo::EMB) p = table + (size_t)__ldg(pa + map.src(m)) * Geo::EMB + (r.i - Geo::FLAT);
    else p = hin + (size_t)m * L + (r.i - Geo::FLAT - Geo::EMB);
    return __ldg(reinterpret_cast<const float4*>(p));
  }
};

// --------------------------------------------------------------------------------------------
// Ape-X dueling network operands (model/apex_value.py:22-41): both streams read
// concat_m = [flatten(a3_m) | emb[previous_action_m]] (K = 3392); rows are already in caller order.
// --------------------------------------------------------------------------------------------
struct CatA {    // K-contiguous rows
  static constexpr bool kContigK = true;
  const float* e;       // [M, 3136]
  const float* table;   // [A, 256]
  const int* pa;        // [M]
  struct Row { const float *pe, *pu; };
  __device__ __forceinline__ Row row(int, int m) const {
    Row r;
    if (m < 0) { r.pe = nullptr; r.pu = nullptr; return r; }
    r.pe = e + (size_t)m * Geo::FLAT;
    r.pu = table + (size_t)__ldg(pa + m) * Geo::EMB;
    return r;
  }
  __device__ __forceinline__ float4 load(const Row& r, int k) const {
    if (r.pe == nullptr) return zero4();
    return __ldg(reinterpret_cast<const float4*>((k < Geo::FLAT) ? r.pe + k : r.pu + (k - Geo::FLAT)));
  }
};
struct CatAT {   // transposed view for dW1 = concat^T dhid1 : index i = feature (contiguous), reduction r = row
  static constexpr bool kContigK = false;
  const float* e;
  const float* table;
  const int* pa;
  struct Row { int i; };
  __device__ __forceinline__ Row row(int, int i) const { Row r; r.i = i; return r; }
  __device__ __forceinline__ float4 load(const Row& r, int m) const {
    if (r.i < 0) return zero4();
    const float* p = (r.i < Geo::FLAT) ? e + (size_t)m * Geo::FLAT + r.i
                                       : table + (size_t)__ldg(pa + m) * Geo::EMB + (r.i - Geo::FLAT);
    return __ldg(reinterpret_cast<const float4*>(p));
  }
};
// Two matrices side by side along N (B(k, n) = n < n0 ? b0[k][n] : b1[k][n - n0]), N-contiguous: the first layers
// of the value and the "mean" stream evaluated by ONE GEMM with N = 2 * 256.
struct DualB {
  static constexpr bool kContigK = false;
  const float* b0; const float* b1; int ldb; int n0;
  struct Row { const float* p; };
  __device__ __forceinline__ Row row(int, int n) const {
    Row r;
    r.p = n < 0 ? nullptr : (n < n0 ? b0 + n : b1 + (n - n0));
    return r;
  }
  __device__ __forceinline__ float4 load(const Row& r, int k) const {
    return r.p ? __ldg(reinterpret_cast<const float4*>(r.p + (size_t)k * ldb)) : zero4();
  }
};
// Two matrices side by side along K: A(m, k) = k < k0 ? a0[m][k] : a1[m][k - k0], K-contiguous, and the matching
// B(k, n) = k < k0 ? w0[n][k] : w1[n][k - k0] (transposed weights): d concat = dhid1_value W1v^T + dhid1_mean W1m^T
// as ONE GEMM with K = 2 * 256.
struct DualA {
  static constexpr bool kContigK = true;
  const float* a0; const float* a1; int lda; int k0;
  struct Row { const float *p0, *p1; };
  __device__ __forceinline__ Row row(int, int m) const {
    Row r;
    if (m < 0) { r.p0 = nullptr; r.p1 = nullptr; return r; }
    r.p0 = a0 + (size_t)m * lda;
    r.p1 = a1 + (size_t)m * lda;
    return r;
  }
  __device__ __forceinline__ float4 load(const Row& r, int k) const {
    if (r.p0 == nullptr) return zero4();
    return __ldg(reinterpret_cast<const float4*>(k < k0 ? r.p0 + k : r.p1 + (k - k0)));
  }
};
struct DualBT {
  static constexpr bool kContigK = true;
  const float* w0; const float* w1; int ldb; int k0;
  struct Row { const float *p0, *p1; };
  __device__ __forceinline__ Row row(int, int n) const {
    Row r;
    if (n < 0) { r.p0 = nullptr; r.p1 = nullptr; return r; }
    r.p0 = w0 + (size_t)n * ldb;
    r.p1 = w1 + (size_t)n * ldb;
    return r;
  }
  __device__ __forceinline__ float4 load(const Row& r, int k) const {
    if (r.p0 == nullptr) return zero4();
    return __ldg(reinterpret_cast<const float4*>(k < k0 ? r.p0 + k : r.p1 + (k - k0)));
  }
};

// --------------------------------------------------------------------------------------------
// Plain strided operands (z = batch index with element strides sz).
// --------------------------------------------------------------------------------------------
struct PlainA {    // A[z][m][k], K-contiguous
  static constexpr bool kContigK = true;
  const float* a; int lda; size_t sz;
  struct Row { const float* p; };
  __device__ __forceinline__ Row row(int z, int m) const { Row r; r.p = m < 0 ? nullptr : a + z * sz + (size_t)m * lda; return r; }
  __device__ __forceinline__ float4 load(const Row& r, int k) const {
    return r.p ? __ldg(reinterpret_cast<const float4*>(r.p + k)) : zero4();
  }
};
struct PlainAT {   // A stored [z][r][i]; GEMM index i contiguous, reduction r
  static constexpr bool kContigK = false;
  const float* a; int lda; size_t sz;
  struct Row { const float* p; };
  __device__ __forceinline__ Row row(int z, int i) const { Row r; r.p = i < 0 ? nullptr : a + z * sz + i; return r; }
  __device__ __forceinline__ float4 load(const Row& r, int rr) const {
    return r.p ? __ldg(reinterpret_cast<const float4*>(r.p + (size_t)rr * lda)) : zero4();
  }
};
struct PlainB {    // B[z][k][n], N-contiguous
  static constexpr bool kContigK = false;
  const float* b; int ldb; size_t sz;
  struct Row { const float* p; };
  __device__ __forceinline__ Row row(int z, int n) const { Row r; r.p = n < 0 ? nullptr : b + z * sz + n; return r; }
  __device__ __forceinline__ float4 load(const Row& r, int k) const {
    return r.p ? __ldg(reinterpret_cast<const float4*>(r.p + (size_t)k * ldb)) : zero4();
  }
};
struct PlainBT {   // B(k, n) = W[z][n][k], K-contiguous (used for dX = dY W^T)
  static constexpr bool kContigK = true;
  const float* b; int ldb; size_t sz;
  struct Row { const float* p; };
  __device__ __forceinline__ Row row(int z, int n) const { Row r; r.p = n < 0 ? nullptr : b + z * sz + (size_t)n * ldb; return r; }
  __device__ __forceinline__ float4 load(const Row& r, int k) const {
    return r.p ? __ldg(reinterpret_cast<const float4*>(r.p + k)) : zero4();
  }
};

// --------------------------------------------------------------------------------------------
// Epilogues
// --------------------------------------------------------------------------------------------
// C[z][m][n] = act(v * scale + bias[z][n])
template <bool RELU, bool BIAS>
struct EpBiasAct {
  static constexpr bool kColSum = false;
  float* c; int ldc; size_t sz;
  const float* bias; size_t sbias;
  float scale;
  Plane16 plane{};   // optional 16-bit plane of c
  template <int V>
  __device__ __forceinline__ void store(int z, int m, int n, const float (&v)[V]) const {
    float o[V];
#pragma unroll
    for (int j = 0; j < V; ++j) {
      float t = v[j] * scale;
      if (BIAS) t += __ldg(bias + z * sbias + n + j);
      o[j] = RELU ? fmaxf(t, 0.f) : t;
    }
    const size_t off = z * sz + (size_t)m * ldc + n;
    if constexpr (V == 4) {
      *reinterpret_cast<float4*>(c + off) = make_float4(o[0], o[1], o[2], o[3]);
      plane.store4(off, o[0], o[1], o[2], o[3]);
    } else {
      c[off] = o[0];
      plane.store1(off, o[0]);
    }
  }
  // hoisted-bias form used by the tensor-core epilogues (epilogue_store_32x32)
  __device__ __forceinline__ float4 bias4(int z, int n) const {
    return BIAS ? __ldg(reinterpret_cast<const float4*>(bias + z * sbias + n)) : zero4();
  }
  __device__ __forceinline__ void store4b(int z, int m, int n, const float (&v)[4], const float4& b) const {
    const float bb[4] = {b.x, b.y, b.z, b.w};
    float o[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float t = v[j] * scale + bb[j];
      o[j] = RELU ? fmaxf(t, 0.f) : t;
    }
    const size_t off = z * sz + (size_t)m * ldc + n;
    *reinterpret_cast<float4*>(c + off) = make_float4(o[0], o[1], o[2], o[3]);
    plane.store4(off, o[0], o[1], o[2], o[3]);
  }
  __device__ __forceinline__ void store_colsum(int, int, float) const {}
};
// x / 255 without the IEEE-division subroutine: nvcc turns `x / 255.0f` into FCHK + a CALL to its slow-path routine that
// cost ~250 cycles per element here (tools/conv1_timeline.py: 32 divisions per thread made the epilogue of a 128x32 tile
// take 11,000 cycles, 80 % of the conv1 kernel).  q = x*r, one FMA residual step: the correctly rounded quotient for all
// finite x outside the denormal range (r = RN(1/255); the residual is exact in FMA arithmetic).
__device__ __forceinline__ float div255(float x) {
  const float r = 1.0f / 255.0f;
  const float q = x * r;
  return fmaf(fmaf(-q, 255.0f, x), r, q);
}
// conv1: the frame bytes are kept as exact integers in the contraction and the /255 of
// agent/impala.py:133 is applied to the accumulator (correctly rounded fp32 quotient, div255), then bias + ReLU.
struct EpConv1 {
  static constexpr bool kColSum = false;
  float* c; int ldc;
  const float* bias;
  Plane16 plane{};   // optional 16-bit plane of c
  template <int V>
  __device__ __forceinline__ void store(int, int m, int n, const float (&v)[V]) const {
    float o[V];
#pragma unroll
    for (int j = 0; j < V; ++j) o[j] = fmaxf(div255(v[j]) + __ldg(bias + n + j), 0.f);
    const size_t off = (size_t)m * ldc + n;
    if constexpr (V == 4) {
      *reinterpret_cast<float4*>(c + off) = make_float4(o[0], o[1], o[2], o[3]);
      plane.store4(off, o[0], o[1], o[2], o[3]);
    } else {
      c[off] = o[0];
      plane.store1(off, o[0]);
    }
  }
  __device__ __forceinline__ float4 bias4(int, int n) const { return __ldg(reinterpret_cast<const float4*>(bias + n)); }
  __device__ __forceinline__ void store4b(int, int m, int n, const float (&v)[4], const float4& b) const {
    const float bb[4] = {b.x, b.y, b.z, b.w};
    float o[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) o[j] = fmaxf(div255(v[j]) + bb[j], 0.f);
    const size_t off = (size_t)m * ldc + n;
    *reinterpret_cast<float4*>(c + off) = make_float4(o[0], o[1], o[2], o[3]);
    plane.store4(off, o[0], o[1], o[2], o[3]);
  }
  __device__ __forceinline__ void store_colsum(int, int, float) const {}
};
// Raw store (split-K partials / batched partial sums): C[z][m][n] = v * scale ; optional column sums
// of B written at row `krow` (the bias-gradient row that follows a [K, N] weight gradient).
template <bool COLSUM>
struct EpRaw {
  static constexpr bool kColSum = COLSUM;
  float* c; int ldc; size_t sz;
  float scale;
  int krow; int nreal;   // nreal < N pads: only n < nreal is stored, with row stride ldc
  template <int V>
  __device__ __forceinline__ void store(int z, int m, int n, const float (&v)[V]) const {
    float* p = c + z * sz + (size_t)m * ldc + n;
    if (V == 4 && n + 3 < nreal && (ldc & 3) == 0) {
      *reinterpret_cast<float4*>(p) = make_float4(v[0] * scale, v[1] * scale, v[2] * scale, v[3] * scale);
    } else {
#pragma unroll
      for (int j = 0; j < V; ++j)
        if (n + j < nreal) p[j] = v[j] * scale;
    }
  }
  __device__ __forceinline__ void store_colsum(int z, int n, float v) const {
    if (n < nreal) c[z * sz + (size_t)krow * ldc + n] = v;
  }
};
// dX with ReLU mask of the forward activation: C[z][m][n] = v * (act[z][m][n] > 0)
struct EpReluMask {
  static constexpr bool kColSum = false;
  float* c; const float* act; int ldc; size_t sz_c; size_t sz_act;
  template <int V>
  __device__ __forceinline__ void store(int z, int m, int n, const float (&v)[V]) const {
    const size_t o = (size_t)m * ldc + n;
    float* pc = c + z * sz_c + o;
    const float* pa = act + z * sz_act + o;
    if constexpr (V == 4) {
      if ((ldc & 3) == 0) {          // n is a multiple of 4 here: 16-byte aligned
        const float4 a = __ldg(reinterpret_cast<const float4*>(pa));
        *reinterpret_cast<float4*>(pc) = make_float4(a.x > 0.f ? v[0] : 0.f, a.y > 0.f ? v[1] : 0.f,
                                                     a.z > 0.f ? v[2] : 0.f, a.w > 0.f ? v[3] : 0.f);
        return;
      }
    }
#pragma unroll
    for (int j = 0; j < V; ++j) pc[j] = (__ldg(pa + j) > 0.f) ? v[j] : 0.f;
  }
  __device__ __forceinline__ void store_colsum(int, int, float) const {}
};
// LSTM input gradient: columns [0,3136) -> d a3 (masked by ReLU of a3), [3136,3392) -> d emb rows.
struct EpLstmDx {
  static constexpr bool kColSum = false;
  float* da3; const float* a3; float* du;
  Plane16 plane{};   // optional 16-bit plane of da3
  template <int V>
  __device__ __forceinline__ void store(int, int m, int n, const float (&v)[V]) const {
    if constexpr (V == 4) {          // FLAT and EMB are multiples of 4: a 4-group never straddles the boundary
      if (n < Geo::FLAT) {
        const size_t o = (size_t)m * Geo::FLAT + n;
        const float4 a = __ldg(reinterpret_cast<const float4*>(a3 + o));
        const float4 d = make_float4(a.x > 0.f ? v[0] : 0.f, a.y > 0.f ? v[1] : 0.f, a.z > 0.f ? v[2] : 0.f,
                                     a.w > 0.f ? v[3] : 0.f);
        *reinterpret_cast<float4*>(da3 + o) = d;
        plane.store4(o, d.x, d.y, d.z, d.w);
      } else {
        *reinterpret_cast<float4*>(du + (size_t)m * Geo::EMB + (n - Geo::FLAT)) = make_float4(v[0], v[1], v[2], v[3]);
      }
      return;
    }
#pragma unroll
    for (int j = 0; j < V; ++j) {
      const int nn = n + j;
      if (nn < Geo::FLAT) {
        const size_t o = (size_t)m * Geo::FLAT + nn;
        const float d = (__ldg(a3 + o) > 0.f) ? v[j] : 0.f;
        da3[o] = d;
        plane.store1(o, d);
      } else {
        du[(size_t)m * Geo::EMB + (nn - Geo::FLAT)] = v[j];
      }
    }
  }
  __device__ __forceinline__ void store_colsum(int, int, float) const {}
};
// Convolution data gradient: row m of parity class z -> pixel (yy*S+py, xx*S+px); masked by ReLU.
template <int IH, int IW, int CI, int S, int RH, int RW>
struct EpConvDx {
  static constexpr bool kColSum = false;
  float* dx; const float* act;
  Plane16 plane{};   // optional 16-bit plane of dx
  template <int V>
  __device__ __forceinline__ void store(int z, int m, int n, const float (&v)[V]) const {
    const int img = m / (RH * RW);
    const int p = m - img * (RH * RW);
    const int yy = p / RW, xx = p - yy * RW;
    const int py = z / S, px = z - py * S;
    const size_t o = ((size_t)(img * IH + yy * S + py) * IW + (xx * S + px)) * CI + n;
    if constexpr (V == 4) {          // CI is a multiple of 4 and n a multiple of 4: 16-byte aligned
      const float4 a = __ldg(reinterpret_cast<const float4*>(act + o));
      const float4 d = make_float4(a.x > 0.f ? v[0] : 0.f, a.y > 0.f ? v[1] : 0.f, a.z > 0.f ? v[2] : 0.f,
                                   a.w > 0.f ? v[3] : 0.f);
      *reinterpret_cast<float4*>(dx + o) = d;
      plane.store4(o, d.x, d.y, d.z, d.w);
    } else {
#pragma unroll
      for (int j = 0; j < V; ++j) {
        const float d = (__ldg(act + o + j) > 0.f) ? v[j] : 0.f;
        dx[o + j] = d;
        plane.store1(o + j, d);
      }
    }
  }
  __device__ __forceinline__ void store_colsum(int, int, float) const {}
};
// The same for the merged-phase GEMM (ConvDgradBMerged): column n = (z, ci).  The 4 columns of a store never straddle
// two classes (CI is a multiple of 4), and the 32 columns of an epilogue block are CI = 32 channels of one pixel.
template <int IH, int IW, int CI, int S, int RH, int RW>
struct EpConvDxMerged {
  static constexpr bool kColSum = false;
  EpConvDx<IH, IW, CI, S, RH, RW> e;
  template <int V>
  __device__ __forceinline__ void store(int, int m, int n, const float (&v)[V]) const {
    e.template store<V>(n / CI, m, n % CI, v);
  }
  __device__ __forceinline__ void store_colsum(int, int, float) const {}
};

}  // namespace drl
