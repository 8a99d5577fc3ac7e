// dev_eq.cuh -- per-RE equalisers shared by the PDCCH and PDSCH kernels (zero forcing: the reference
// leaves decoder_type = 0, SURVEY.md App. B.7), the zero-denominator rule they share with the PUSCH kernel, and the int16 soft
// demapper with descrambling of the PDSCH and PUSCH kernels.  Operation order mirrors the CPU oracles exactly.
#pragma once
#include "dev_common.cuh"

struct SfView {
  const float2* y[2];      // per antenna [14*nsc]
  const float2* pil[2][2]; // [port][ant] -> smoothed CRS estimates [NPILSYM][2 nof_prb] (chest_kernel); the per-RE estimate is interpolated here
};

// Channel estimate of (port p, antenna a) at resource element idx = l * nsc + k: linear interpolation in frequency between the two
// neighbouring pilots of the pilot symbols around l, then in time -- the expression chest_interp_kernel (k_frontend.cu) evaluates when the
// whole grid is asked for, so the value is bit-identical to ltephy_tap(LTEPHY_TAP_CE).  Fusing it into the equalisers saves the 537 KB per
// subframe round trip of the interpolated grid through HBM.
__device__ __forceinline__ float2 ce_f_interp(const DevCell& c, const float2* sm, uint32_t np, uint32_t off, uint32_t k)
{
  int m = ((int)k - (int)off) / 6;
  if ((int)k < (int)off) m = 0;
  if (m > (int)np - 2) m = (int)np - 2;
  const int    j  = (int)k - (6 * m + (int)off);
  const float  cc = c.interp_c[j + 5];
  const float2 A = sm[m], B = sm[m + 1];
  return make_float2(A.x + (B.x - A.x) * cc, A.y + (B.y - A.y) * cc);
}
__device__ __forceinline__ float2 ce_at(const DevCell& c, const float2* pil, uint32_t p, uint32_t l, uint32_t k)
{
  const uint32_t np = 2 * c.nof_prb, ia = c.t_ia[l], ib = c.t_ib[l];
  const float    t  = c.t_frac[l];
  const float2   A = ce_f_interp(c, pil + ia * np, np, c.crs_off[p][ia & 1], k);
  const float2   B = ce_f_interp(c, pil + ib * np, np, c.crs_off[p][ib & 1], k);
  if (l < 11) return make_float2(A.x + (B.x - A.x) * t, A.y + (B.y - A.y) * t);
  return make_float2(B.x + (B.x - A.x) * t, B.y + (B.y - A.y) * t);
}
__device__ __forceinline__ float2 h_at(const DevCell& c, const SfView& v, uint32_t p, uint32_t a, uint32_t idx)
{
  const uint32_t l = idx / c.nsc;
  return ce_at(c, v.pil[p][a], p, l, idx - l * c.nsc);
}

// numerator / denominator of an equaliser, with an exactly zero denominator (no channel at all: a zero-filled capture, a dead antenna, a singular
// 2x2) giving 0 instead of 0/0 = NaN, so that the RE becomes an erasure (LLR 0) -- DESIGN.md section 2.  Every other quotient is unchanged.
__device__ __forceinline__ float eq_div(float n, float d) { return d == 0.0f ? 0.0f : n / d; }

// ---- int16 soft demodulation (srsran_demod_soft_demodulate_s: scales 100*sqrt2 / 400 / 700 / 1000) and descrambling
__device__ __forceinline__ short f2s(float v)
{
  if (isnan(v)) return 0; // fmaxf would turn NaN into -32767, a full-confidence bit
  v = fminf(fmaxf(v, -32767.0f), 32767.0f);
  return (short)(int)v; // truncation toward zero
}
__device__ __forceinline__ int iabs(int v) { return v < 0 ? -v : v; }
__device__ __forceinline__ void demod_s(float2 x, uint32_t qm, short* z)
{
  if (qm == 2) {
    const float s = 141.421356f;
    z[0] = (short)-f2s(x.x * s), z[1] = (short)-f2s(x.y * s);
  } else if (qm == 4) {
    const int yr = f2s(x.x * 400.0f), yi = f2s(x.y * 400.0f);
    z[0] = (short)-yr, z[1] = (short)-yi;
    z[2] = (short)(iabs(yr) - 252), z[3] = (short)(iabs(yi) - 252);
  } else if (qm == 6) {
    const int yr = f2s(x.x * 700.0f), yi = f2s(x.y * 700.0f);
    z[0] = (short)-yr, z[1] = (short)-yi;
    z[2] = (short)(iabs(yr) - 432), z[3] = (short)(iabs(yi) - 432);
    z[4] = (short)(iabs(z[2]) - 216), z[5] = (short)(iabs(z[3]) - 216);
  } else { // 256QAM (on the PUSCH: third attempt of PUSCH_Decoder::decode, reference src/src/UL_Sniffer_PUSCH.cc:508-520)
    const int yr = f2s(x.x * 1000.0f), yi = f2s(x.y * 1000.0f);
    z[0] = (short)-yr, z[1] = (short)-yi;
    z[2] = (short)(iabs(yr) - 613), z[3] = (short)(iabs(yi) - 613);
    z[4] = (short)(iabs(z[2]) - 306), z[5] = (short)(iabs(z[3]) - 306);
    z[6] = (short)(iabs(z[4]) - 153), z[7] = (short)(iabs(z[5]) - 153);
  }
}
// The Qm soft bits of symbol x * scl: demodulate, flip the sign of bit b where bit b0 + b of the sequence seq is set (Qm bits taken from a
// 64-bit window), store Qm / 2 packed int16 pairs at out.  An exactly zero x is an erasure (DESIGN.md section 2): LLR 0.  The zero test is on
// x, before the scale, as in the oracles: a subnormal x that scl rounds to zero still demodulates.  Two conditions make the accesses safe:
// out is 4-byte aligned because Qm is even and alloc_codeword (ltephy_capi.cu) rounds every codeword's soft-bit offset to 8, and the
// window's second word lies inside the pool because alloc_codeword reserves one word past every codeword's sequence.
__device__ __forceinline__ void soft_bits(float2 x, float scl, uint32_t qm, const uint32_t* __restrict__ seq, uint32_t b0, short* __restrict__ out)
{
  short z[8] = {0, 0, 0, 0, 0, 0, 0, 0};
  if (x.x != 0.0f || x.y != 0.0f) demod_s(make_float2(x.x * scl, x.y * scl), qm, z);
  const uint32_t           w0  = b0 >> 5;
  const unsigned long long win = ((unsigned long long)seq[w0] | ((unsigned long long)seq[w0 + 1] << 32)) >> (b0 & 31u);
  uint32_t*                o   = reinterpret_cast<uint32_t*>(out);
#pragma unroll
  for (uint32_t i = 0; i < 8; i += 2) {
    if (i >= qm) break;
    const int a = ((win >> i) & 1ull) ? -(int)z[i] : (int)z[i], b = ((win >> (i + 1)) & 1ull) ? -(int)z[i + 1] : (int)z[i + 1];
    o[i >> 1]   = ((uint32_t)a & 0xFFFFu) | ((uint32_t)b << 16);
  }
}

__device__ __forceinline__ float2 eq_port0(const DevCell& c, const SfView& v, uint32_t idx)
{
  float nr = 0.0f, ni = 0.0f, den = 0.0f;
  for (uint32_t a = 0; a < c.nof_rx; a++) {
    const float2 y = v.y[a][idx], h = h_at(c, v, 0, a, idx);
    nr  = nr + (y.x * h.x + y.y * h.y);
    ni  = ni + (y.y * h.x - y.x * h.y);
    den = den + (h.x * h.x + h.y * h.y);
  }
  return make_float2(eq_div(nr, den), eq_div(ni, den));
}
__device__ __forceinline__ void eq_sfbc(const DevCell& c, const SfView& v, uint32_t i0, uint32_t i1, float2& x0, float2& x1)
{
  float n0r = 0.0f, n0i = 0.0f, n1r = 0.0f, n1i = 0.0f, d0 = 0.0f, d1 = 0.0f;
  for (uint32_t a = 0; a < c.nof_rx; a++) {
    const float2 r0 = v.y[a][i0], r1 = v.y[a][i1];
    const float2 h00 = h_at(c, v, 0, a, i0), h01 = h_at(c, v, 0, a, i1), h10 = h_at(c, v, 1, a, i0), h11 = h_at(c, v, 1, a, i1);
    n0r = n0r + ((h00.x * r0.x + h00.y * r0.y) + (h11.x * r1.x + h11.y * r1.y));
    n0i = n0i + ((h00.x * r0.y - h00.y * r0.x) + (h11.y * r1.x - h11.x * r1.y));
    n1r = n1r + ((h01.x * r1.x + h01.y * r1.y) - (h10.x * r0.x + h10.y * r0.y));
    n1i = n1i + ((h01.x * r1.y - h01.y * r1.x) - (h10.y * r0.x - h10.x * r0.y));
    d0  = d0 + ((h00.x * h00.x + h00.y * h00.y) + (h11.x * h11.x + h11.y * h11.y));
    d1  = d1 + ((h01.x * h01.x + h01.y * h01.y) + (h10.x * h10.x + h10.y * h10.y));
  }
  const float s2 = 1.41421354f;
  x0             = make_float2(eq_div(n0r, d0) * s2, eq_div(n0i, d0) * s2);
  x1             = make_float2(eq_div(n1r, d1) * s2, eq_div(n1i, d1) * s2);
}
// closed-loop spatial multiplexing, 2 CRS ports (36.211 Table 6.3.4.2.3-1): w = second precoder entry
__device__ __forceinline__ float2 spmux_w(uint32_t nof_layers, uint32_t pmi)
{
  if (nof_layers == 1) return (pmi & 3u) == 0 ? make_float2(1.f, 0.f) : (pmi & 3u) == 1 ? make_float2(-1.f, 0.f) : (pmi & 3u) == 2 ? make_float2(0.f, 1.f) : make_float2(0.f, -1.f);
  return (pmi & 1u) ? make_float2(0.f, 1.f) : make_float2(1.f, 0.f);
}
__device__ __forceinline__ float2 eq_spmux1(const DevCell& c, const SfView& v, uint32_t idx, float2 w)
{
  float nr = 0.0f, ni = 0.0f, den = 0.0f;
  for (uint32_t a = 0; a < c.nof_rx; a++) {
    const float2 y = v.y[a][idx], h0 = h_at(c, v, 0, a, idx), h1 = h_at(c, v, 1, a, idx);
    const float2 e = make_float2(h0.x + (w.x * h1.x - w.y * h1.y), h0.y + (w.x * h1.y + w.y * h1.x));
    nr  = nr + (e.x * y.x + e.y * y.y);
    ni  = ni + (e.x * y.y - e.y * y.x);
    den = den + (e.x * e.x + e.y * e.y);
  }
  const float s2 = 1.41421354f;
  return make_float2(eq_div(nr, den) * s2, eq_div(ni, den) * s2);
}
// x = 2 E^-1 r, E rows = rx antennas, columns = layers
__device__ __forceinline__ void zf2x2(float2 e00, float2 e01, float2 e10, float2 e11, float2 r0, float2 r1, float2& x0, float2& x1)
{
  const float2 det = make_float2((e00.x * e11.x - e00.y * e11.y) - (e01.x * e10.x - e01.y * e10.y),
                                 (e00.x * e11.y + e00.y * e11.x) - (e01.x * e10.y + e01.y * e10.x));
  const float2 a0  = make_float2((e11.x * r0.x - e11.y * r0.y) - (e01.x * r1.x - e01.y * r1.y),
                                 (e11.x * r0.y + e11.y * r0.x) - (e01.x * r1.y + e01.y * r1.x));
  const float2 a1  = make_float2((e00.x * r1.x - e00.y * r1.y) - (e10.x * r0.x - e10.y * r0.y),
                                 (e00.x * r1.y + e00.y * r1.x) - (e10.x * r0.y + e10.y * r0.x));
  const float dd = det.x * det.x + det.y * det.y;
  x0 = make_float2(eq_div(a0.x * det.x + a0.y * det.y, dd) * 2.0f, eq_div(a0.y * det.x - a0.x * det.y, dd) * 2.0f);
  x1 = make_float2(eq_div(a1.x * det.x + a1.y * det.y, dd) * 2.0f, eq_div(a1.y * det.x - a1.x * det.y, dd) * 2.0f);
}
__device__ __forceinline__ void eq_spmux2(const DevCell& c, const SfView& v, uint32_t idx, float2 w, float2& x0, float2& x1)
{
  const float2 h00 = h_at(c, v, 0, 0, idx), h10 = h_at(c, v, 0, 1, idx), h01 = h_at(c, v, 1, 0, idx), h11 = h_at(c, v, 1, 1, idx);
  const float2 w0 = make_float2(w.x * h01.x - w.y * h01.y, w.x * h01.y + w.y * h01.x);
  const float2 w1 = make_float2(w.x * h11.x - w.y * h11.y, w.x * h11.y + w.y * h11.x);
  zf2x2(make_float2(h00.x + w0.x, h00.y + w0.y), make_float2(h00.x - w0.x, h00.y - w0.y), make_float2(h10.x + w1.x, h10.y + w1.y),
        make_float2(h10.x - w1.x, h10.y - w1.y), v.y[0][idx], v.y[1][idx], x0, x1);
}
__device__ __forceinline__ void eq_cdd(const DevCell& c, const SfView& v, uint32_t idx, bool odd, float2& x0, float2& x1)
{
  const float2 r0 = v.y[0][idx], r1 = v.y[1][idx];
  const float2 h00 = h_at(c, v, 0, 0, idx), h10 = h_at(c, v, 0, 1, idx), h01 = h_at(c, v, 1, 0, idx), h11 = h_at(c, v, 1, 1, idx);
  const float  s = odd ? -1.0f : 1.0f;
  const float2 e00 = make_float2(h00.x + s * h01.x, h00.y + s * h01.y), e01 = make_float2(h00.x - s * h01.x, h00.y - s * h01.y);
  const float2 e10 = make_float2(h10.x + s * h11.x, h10.y + s * h11.y), e11 = make_float2(h10.x - s * h11.x, h10.y - s * h11.y);
  const float2 det = make_float2((e00.x * e11.x - e00.y * e11.y) - (e01.x * e10.x - e01.y * e10.y),
                                 (e00.x * e11.y + e00.y * e11.x) - (e01.x * e10.y + e01.y * e10.x));
  const float2 a0  = make_float2((e11.x * r0.x - e11.y * r0.y) - (e01.x * r1.x - e01.y * r1.y),
                                 (e11.x * r0.y + e11.y * r0.x) - (e01.x * r1.y + e01.y * r1.x));
  const float2 a1  = make_float2((e00.x * r1.x - e00.y * r1.y) - (e10.x * r0.x - e10.y * r0.y),
                                 (e00.x * r1.y + e00.y * r1.x) - (e10.x * r0.y + e10.y * r0.x));
  const float dd = det.x * det.x + det.y * det.y;
  x0 = make_float2(eq_div(a0.x * det.x + a0.y * det.y, dd) * 2.0f, eq_div(a0.y * det.x - a0.x * det.y, dd) * 2.0f);
  x1 = make_float2(eq_div(a1.x * det.x + a1.y * det.y, dd) * 2.0f, eq_div(a1.y * det.x - a1.x * det.y, dd) * 2.0f);
}
__device__ __forceinline__ SfView make_view(const DevCell& c, const float2* sym, const float2* pil, uint32_t sf)
{
  SfView         v;
  const uint32_t g = 14 * c.nsc, gp = NPILSYM * 2 * c.nof_prb;
  for (uint32_t a = 0; a < 2; a++) {
    v.y[a] = sym + ((size_t)sf * c.nof_rx + (a < c.nof_rx ? a : 0)) * g;
    for (uint32_t p = 0; p < 2; p++)
      v.pil[p][a] = pil + (((size_t)sf * c.nof_ports + (p < c.nof_ports ? p : 0)) * c.nof_rx + (a < c.nof_rx ? a : 0)) * gp;
  }
  return v;
}
