/*
 * oracle/kquants_port.c — TEST INFRASTRUCTURE, NOT PRODUCT CODE.
 *
 * A plain-C restatement ("port") of the reference's CPU algorithm for the quantized decode
 * hot path.  It exists only so that tests/, __graft_entry__.smoke() and bench.py's
 * cpu_baseline / --impl reference legs can check the CUDA path; nothing under
 * prima.cpp_b200/ may link, import or call it.
 *
 * Parity pin: every function here is checked (tests/test_oracle_port.py) against
 *   (1) the real reference compiled into oracle/_ref/, through its outputs recorded in tests/golden/reference_golden.npz, and
 *   (2) committed golden vectors in tests/golden/*.npz generated from that same compiled
 *       reference by tests/golden/make_golden.py.
 *
 * Each function cites the reference file:line it follows (paths relative to the reference source tree).
 * Written from the algorithm description; scalar form only (SIMD paths of the reference are
 * integer-identical and differ only in fp32 summation order).
 */
#define _GNU_SOURCE
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#define QK_K 256

/* ---- block layouts: ggml/src/ggml-common.h:143-170, 173-204, 286-335 (byte-for-byte wire format) ---- */
#pragma pack(push, 1)
typedef struct { uint16_t d; uint8_t qs[16]; } blk_q4_0;                                          /* 18 B */
typedef struct { uint16_t d, m; uint8_t qs[16]; } blk_q4_1;                                       /* 20 B */
typedef struct { uint16_t d; uint8_t qh[4]; uint8_t qs[16]; } blk_q5_0;                           /* 22 B */
typedef struct { uint16_t d, dmin; uint8_t scales[12]; uint8_t qs[128]; } blk_q4_K;              /* 144 B */
typedef struct { uint16_t d, dmin; uint8_t scales[12]; uint8_t qh[32]; uint8_t qs[128]; } blk_q5_K; /* 176 B */
typedef struct { uint8_t ql[128]; uint8_t qh[64]; int8_t scales[16]; uint16_t d; } blk_q6_K;     /* 210 B */
typedef struct { uint16_t d; int8_t qs[32]; } blk_q8_0;                                          /* 34 B */
typedef struct { uint16_t d, m; uint8_t qh[4]; uint8_t qs[16]; } blk_q5_1;                       /* 24 B */
typedef struct { uint16_t d, s; int8_t qs[32]; } blk_q8_1;                                       /* 36 B */
typedef struct { float d; int8_t qs[256]; int16_t bsums[16]; } blk_q8_K;                         /* 292 B */
#pragma pack(pop)

enum { T_F32 = 0, T_F16 = 1, T_Q4_0 = 2, T_Q4_1 = 3, T_Q5_0 = 6, T_Q5_1 = 7, T_Q8_0 = 8, T_Q4_K = 12, T_Q5_K = 13, T_Q6_K = 14 }; /* ggml.h:356-395 */

/* ---- fp16 <-> fp32, IEEE round-to-nearest-even (ggml-impl.h GGML_FP16_TO_FP32 / FP32_TO_FP16) ---- */
float port_fp16_to_fp32(uint16_t h) {
    uint32_t sign = (uint32_t)(h & 0x8000) << 16;
    uint32_t exp  = (h >> 10) & 0x1f;
    uint32_t man  = h & 0x3ff;
    uint32_t bits;
    if (exp == 0) {
        if (man == 0) { bits = sign; }
        else {
            int e = -1;
            do { man <<= 1; e++; } while (!(man & 0x400));
            bits = sign | ((uint32_t)(127 - 15 - e) << 23) | ((man & 0x3ff) << 13);
        }
    } else if (exp == 31) {
        bits = sign | 0x7f800000u | (man << 13);
    } else {
        bits = sign | ((exp + 112) << 23) | (man << 13);
    }
    float f; memcpy(&f, &bits, 4); return f;
}

uint16_t port_fp32_to_fp16(float f) {
    uint32_t x; memcpy(&x, &f, 4);
    uint32_t sign = (x >> 16) & 0x8000;
    uint32_t ax = x & 0x7fffffffu;
    if (ax >= 0x7f800000u) return (uint16_t)(sign | 0x7c00 | (ax > 0x7f800000u ? 0x200 : 0));
    if (ax >= 0x477ff000u) return (uint16_t)(sign | 0x7c00);          /* overflow -> inf (65520 rounds up) */
    if (ax < 0x33000001u) return (uint16_t)sign;                      /* < 2^-25 (or == 2^-25 tie -> 0) */
    int32_t e = (int32_t)(ax >> 23) - 127;
    uint32_t m = (ax & 0x7fffffu) | 0x800000u;
    int shift;
    uint32_t base;
    if (e < -14) { shift = 13 + (-14 - e); base = 0; }
    else         { shift = 13; base = (uint32_t)(e + 15) << 10; m &= 0x7fffffu; }
    uint32_t q = m >> shift;
    uint32_t rem = m & ((1u << shift) - 1);
    uint32_t half = 1u << (shift - 1);
    if (rem > half || (rem == half && (q & 1))) q++;
    return (uint16_t)(sign | (base + q));   /* mantissa carry propagates into the exponent field */
}

/* ggml-quants.c:1639-1644 — round-half-even through the 1.5*2^23 magic constant */
static inline int nearest_int(float fval) {
    float val = fval + 12582912.f;
    int i; memcpy(&i, &val, sizeof(int));
    return (i & 0x007fffff) - 0x00400000;
}

/* ggml-quants.c:1898-1905 */
static inline void get_scale_min_k4(int j, const uint8_t *q, uint8_t *d, uint8_t *m) {
    if (j < 4) { *d = q[j] & 63; *m = q[j + 4] & 63; }
    else {
        *d = (q[j + 4] & 0xF) | ((q[j - 4] >> 6) << 4);
        *m = (q[j + 4] >> 4) | ((q[j] >> 6) << 4);
    }
}

/* ---------------- dequantization (ggml-quants.c:2555-2577, 2763-2788, 2977-3006, 1616-1634, 1589-1613, 1522-1580) ----------------
 * In the 32-element blocks element j < 16 is the low nibble of qs[j], element j + 16 its high nibble; the fifth bit of element j is
 * bit j of qh. */
void port_dequantize_row_q4_K(const void *vx, float *y, int64_t k) {
    const blk_q4_K *x = (const blk_q4_K *)vx;
    for (int64_t i = 0; i < k / QK_K; i++) {
        const uint8_t *q = x[i].qs;
        const float d = port_fp16_to_fp32(x[i].d), mn = port_fp16_to_fp32(x[i].dmin);
        int is = 0; uint8_t sc, m;
        for (int j = 0; j < QK_K; j += 64) {
            get_scale_min_k4(is + 0, x[i].scales, &sc, &m); const float d1 = d * sc, m1 = mn * m;
            get_scale_min_k4(is + 1, x[i].scales, &sc, &m); const float d2 = d * sc, m2 = mn * m;
            for (int l = 0; l < 32; ++l) *y++ = d1 * (q[l] & 0xF) - m1;
            for (int l = 0; l < 32; ++l) *y++ = d2 * (q[l] >> 4) - m2;
            q += 32; is += 2;
        }
    }
}

void port_dequantize_row_q5_K(const void *vx, float *y, int64_t k) {
    const blk_q5_K *x = (const blk_q5_K *)vx;
    for (int64_t i = 0; i < k / QK_K; i++) {
        const uint8_t *ql = x[i].qs, *qh = x[i].qh;
        const float d = port_fp16_to_fp32(x[i].d), mn = port_fp16_to_fp32(x[i].dmin);
        int is = 0; uint8_t sc, m; uint8_t u1 = 1, u2 = 2;
        for (int j = 0; j < QK_K; j += 64) {
            get_scale_min_k4(is + 0, x[i].scales, &sc, &m); const float d1 = d * sc, m1 = mn * m;
            get_scale_min_k4(is + 1, x[i].scales, &sc, &m); const float d2 = d * sc, m2 = mn * m;
            for (int l = 0; l < 32; ++l) *y++ = d1 * ((ql[l] & 0xF) + (qh[l] & u1 ? 16 : 0)) - m1;
            for (int l = 0; l < 32; ++l) *y++ = d2 * ((ql[l] >> 4) + (qh[l] & u2 ? 16 : 0)) - m2;
            ql += 32; is += 2; u1 <<= 2; u2 <<= 2;
        }
    }
}

void port_dequantize_row_q6_K(const void *vx, float *y, int64_t k) {
    const blk_q6_K *x = (const blk_q6_K *)vx;
    for (int64_t i = 0; i < k / QK_K; i++) {
        const float d = port_fp16_to_fp32(x[i].d);
        const uint8_t *ql = x[i].ql, *qh = x[i].qh; const int8_t *sc = x[i].scales;
        for (int n = 0; n < QK_K; n += 128) {
            for (int l = 0; l < 32; ++l) {
                int is = l / 16;
                const int8_t q1 = (int8_t)((ql[l +  0] & 0xF) | (((qh[l] >> 0) & 3) << 4)) - 32;
                const int8_t q2 = (int8_t)((ql[l + 32] & 0xF) | (((qh[l] >> 2) & 3) << 4)) - 32;
                const int8_t q3 = (int8_t)((ql[l +  0] >> 4) | (((qh[l] >> 4) & 3) << 4)) - 32;
                const int8_t q4 = (int8_t)((ql[l + 32] >> 4) | (((qh[l] >> 6) & 3) << 4)) - 32;
                y[l +  0] = d * sc[is + 0] * q1;
                y[l + 32] = d * sc[is + 2] * q2;
                y[l + 64] = d * sc[is + 4] * q3;
                y[l + 96] = d * sc[is + 6] * q4;
            }
            y += 128; ql += 64; qh += 32; sc += 8;
        }
    }
}

void port_dequantize_row_q8_0(const void *vx, float *y, int64_t k) {
    const blk_q8_0 *x = (const blk_q8_0 *)vx;
    for (int64_t i = 0; i < k / 32; i++) {
        const float d = port_fp16_to_fp32(x[i].d);
        for (int j = 0; j < 32; ++j) y[i * 32 + j] = x[i].qs[j] * d;
    }
}

void port_dequantize_row_q5_1(const void *vx, float *y, int64_t k) {
    const blk_q5_1 *x = (const blk_q5_1 *)vx;
    for (int64_t i = 0; i < k / 32; i++) {
        const float d = port_fp16_to_fp32(x[i].d), m = port_fp16_to_fp32(x[i].m);
        uint32_t qh; memcpy(&qh, x[i].qh, 4);
        for (int j = 0; j < 16; ++j) {
            const uint8_t xh_0 = ((qh >> (j + 0)) << 4) & 0x10;
            const uint8_t xh_1 = ((qh >> (j + 12))) & 0x10;
            const int x0 = (x[i].qs[j] & 0x0F) | xh_0;
            const int x1 = (x[i].qs[j] >> 4) | xh_1;
            y[i * 32 + j] = x0 * d + m;
            y[i * 32 + j + 16] = x1 * d + m;
        }
    }
}

/* ggml-quants.c:1522-1540 */
void port_dequantize_row_q4_0(const void *vx, float *y, int64_t k) {
    const blk_q4_0 *x = (const blk_q4_0 *)vx;
    for (int64_t i = 0; i < k / 32; i++) {
        const float d = port_fp16_to_fp32(x[i].d);
        for (int j = 0; j < 16; ++j) {
            const int x0 = (x[i].qs[j] & 0x0F) - 8;
            const int x1 = (x[i].qs[j] >> 4) - 8;
            y[i * 32 + j] = x0 * d;
            y[i * 32 + j + 16] = x1 * d;
        }
    }
}

/* ggml-quants.c:1542-1561 */
void port_dequantize_row_q4_1(const void *vx, float *y, int64_t k) {
    const blk_q4_1 *x = (const blk_q4_1 *)vx;
    for (int64_t i = 0; i < k / 32; i++) {
        const float d = port_fp16_to_fp32(x[i].d), m = port_fp16_to_fp32(x[i].m);
        for (int j = 0; j < 16; ++j) {
            const int x0 = x[i].qs[j] & 0x0F;
            const int x1 = x[i].qs[j] >> 4;
            y[i * 32 + j] = x0 * d + m;
            y[i * 32 + j + 16] = x1 * d + m;
        }
    }
}

/* ggml-quants.c:1563-1586 */
void port_dequantize_row_q5_0(const void *vx, float *y, int64_t k) {
    const blk_q5_0 *x = (const blk_q5_0 *)vx;
    for (int64_t i = 0; i < k / 32; i++) {
        const float d = port_fp16_to_fp32(x[i].d);
        uint32_t qh; memcpy(&qh, x[i].qh, 4);
        for (int j = 0; j < 16; ++j) {
            const uint8_t xh_0 = ((qh >> (j + 0)) << 4) & 0x10;
            const uint8_t xh_1 = ((qh >> (j + 12))) & 0x10;
            const int32_t x0 = ((x[i].qs[j] & 0x0F) | xh_0) - 16;
            const int32_t x1 = ((x[i].qs[j] >> 4) | xh_1) - 16;
            y[i * 32 + j] = x0 * d;
            y[i * 32 + j + 16] = x1 * d;
        }
    }
}

int64_t port_row_size(int type, int64_t k) {   /* ggml_row_size, ggml.c type-traits table :732-1100 */
    switch (type) {
        case T_F32: return k * 4;
        case T_F16: return k * 2;
        case T_Q4_K: return k / 256 * 144;
        case T_Q5_K: return k / 256 * 176;
        case T_Q6_K: return k / 256 * 210;
        case T_Q8_0: return k / 32 * 34;
        case T_Q5_1: return k / 32 * 24;
        case T_Q4_0: return k / 32 * 18;
        case T_Q4_1: return k / 32 * 20;
        case T_Q5_0: return k / 32 * 22;
    }
    return -1;
}

void port_dequantize_row(int type, const void *vx, float *y, int64_t k) {
    switch (type) {
        case T_Q4_K: port_dequantize_row_q4_K(vx, y, k); break;
        case T_Q5_K: port_dequantize_row_q5_K(vx, y, k); break;
        case T_Q6_K: port_dequantize_row_q6_K(vx, y, k); break;
        case T_Q8_0: port_dequantize_row_q8_0(vx, y, k); break;
        case T_Q5_1: port_dequantize_row_q5_1(vx, y, k); break;
        case T_Q4_0: port_dequantize_row_q4_0(vx, y, k); break;
        case T_Q4_1: port_dequantize_row_q4_1(vx, y, k); break;
        case T_Q5_0: port_dequantize_row_q5_0(vx, y, k); break;
        case T_F32:  memcpy(y, vx, (size_t)k * 4); break;
        case T_F16:  for (int64_t i = 0; i < k; i++) y[i] = port_fp16_to_fp32(((const uint16_t *)vx)[i]); break;
    }
}

/* ---------------- activation quantization ---------------- */
/* ggml-quants.c:3785-3822 quantize_row_q8_K_ref (the CPU backend's from_float for vec_dot_type Q8_K) */
void port_quantize_row_q8_K(const float *x, void *vy, int64_t k) {
    blk_q8_K *y = (blk_q8_K *)vy;
    for (int64_t i = 0; i < k / QK_K; i++) {
        float max = 0, amax = 0;
        for (int j = 0; j < QK_K; ++j) { float ax = fabsf(x[j]); if (ax > amax) { amax = ax; max = x[j]; } }
        if (!amax) { y[i].d = 0; memset(y[i].qs, 0, QK_K); memset(y[i].bsums, 0, 32); x += QK_K; continue; }
        const float iscale = -127.f / max;
        for (int j = 0; j < QK_K; ++j) { int v = nearest_int(iscale * x[j]); y[i].qs[j] = (int8_t)(v < 127 ? v : 127); }
        for (int j = 0; j < QK_K / 16; ++j) {
            int sum = 0;
            for (int ii = 0; ii < 16; ++ii) sum += y[i].qs[j * 16 + ii];
            y[i].bsums[j] = (int16_t)sum;
        }
        y[i].d = 1 / iscale;
        x += QK_K;
    }
}
/* NOTE: the reference leaves bsums of an all-zero block untouched (garbage from wdata); they are
 * multiplied by d == 0 afterwards, so zeroing them here is result-identical. */

/* ggml-quants.c:873-1157 quantize_row_q8_0, AVX2 branch (:943-1010): d = max/127 stored fp16,
 * id = 127/max, round-to-nearest-EVEN (_mm256_round_ps).  The scalar _ref (:848-872) uses 1/d and
 * roundf (half away); the x86 oracle box runs the AVX2 branch, so that is what is restated. */
void port_quantize_row_q8_0(const float *x, void *vy, int64_t k) {
    blk_q8_0 *y = (blk_q8_0 *)vy;
    for (int64_t i = 0; i < k / 32; i++) {
        float amax = 0.0f;
        for (int j = 0; j < 32; j++) { float v = fabsf(x[i * 32 + j]); if (v > amax) amax = v; }
        const float d = amax / 127.f;
        const float id = (amax != 0.0f) ? 127.f / amax : 0.0f;
        y[i].d = port_fp32_to_fp16(d);
        for (int j = 0; j < 32; ++j) y[i].qs[j] = (int8_t)nearbyintf(x[i * 32 + j] * id);
    }
}

/* ggml-quants.c:1195-1330 quantize_row_q8_1, AVX2 branch: as q8_0 plus s = fp16(d * sum(q)) */
void port_quantize_row_q8_1(const float *x, void *vy, int64_t k) {
    blk_q8_1 *y = (blk_q8_1 *)vy;
    for (int64_t i = 0; i < k / 32; i++) {
        float amax = 0.0f;
        for (int j = 0; j < 32; j++) { float v = fabsf(x[i * 32 + j]); if (v > amax) amax = v; }
        const float d = amax / 127.f;
        const float id = (amax != 0.0f) ? 127.f / amax : 0.0f;
        y[i].d = port_fp32_to_fp16(d);
        int sum = 0;
        for (int j = 0; j < 32; ++j) { int q = (int)nearbyintf(x[i * 32 + j] * id); y[i].qs[j] = (int8_t)q; sum += q; }
        y[i].s = port_fp32_to_fp16(d * sum);
    }
}

/* ---------------- dot products (scalar forms) ---------------- */
/* ggml-quants.c:8222-8277 */
float port_vec_dot_q4_K_q8_K(int n, const void *vx, const void *vy) {
    const blk_q4_K *x = (const blk_q4_K *)vx; const blk_q8_K *y = (const blk_q8_K *)vy;
    float sums[8] = {0}; float sumf = 0;
    for (int i = 0; i < n / QK_K; ++i) {
        int32_t aux32[8] = {0};
        int8_t aux8[QK_K];
        const uint8_t *q4 = x[i].qs; int8_t *a = aux8;
        for (int j = 0; j < QK_K / 64; ++j) {
            for (int l = 0; l < 32; ++l) a[l] = (int8_t)(q4[l] & 0xF);
            a += 32;
            for (int l = 0; l < 32; ++l) a[l] = (int8_t)(q4[l] >> 4);
            a += 32; q4 += 32;
        }
        uint8_t scales[8], mins[8];
        for (int j = 0; j < 8; j++) get_scale_min_k4(j, x[i].scales, &scales[j], &mins[j]);
        int sumi = 0;
        for (int j = 0; j < QK_K / 16; ++j) sumi += y[i].bsums[j] * mins[j / 2];
        const int8_t *q8 = y[i].qs; a = aux8;
        for (int j = 0; j < QK_K / 32; ++j) {
            int32_t scale = scales[j];
            for (int g = 0; g < 4; g++) { for (int l = 0; l < 8; ++l) aux32[l] += scale * (q8[l] * a[l]); q8 += 8; a += 8; }
        }
        const float d = port_fp16_to_fp32(x[i].d) * y[i].d;
        for (int l = 0; l < 8; ++l) sums[l] += d * aux32[l];
        const float dmin = port_fp16_to_fp32(x[i].dmin) * y[i].d;
        sumf -= dmin * sumi;
    }
    for (int l = 0; l < 8; ++l) sumf += sums[l];
    return sumf;
}

/* ggml-quants.c:8854-8916 */
float port_vec_dot_q5_K_q8_K(int n, const void *vx, const void *vy) {
    const blk_q5_K *x = (const blk_q5_K *)vx; const blk_q8_K *y = (const blk_q8_K *)vy;
    float sums[8] = {0}; float sumf = 0;
    for (int i = 0; i < n / QK_K; ++i) {
        int32_t aux32[8] = {0};
        int8_t aux8[QK_K];
        const uint8_t *q4 = x[i].qs, *hm = x[i].qh; int8_t *a = aux8; uint8_t m = 1;
        for (int j = 0; j < QK_K / 64; ++j) {
            for (int l = 0; l < 32; ++l) a[l] = (int8_t)((q4[l] & 0xF) + (hm[l] & m ? 16 : 0));
            a += 32; m <<= 1;
            for (int l = 0; l < 32; ++l) a[l] = (int8_t)((q4[l] >> 4) + (hm[l] & m ? 16 : 0));
            a += 32; m <<= 1; q4 += 32;
        }
        uint8_t scales[8], mins[8];
        for (int j = 0; j < 8; j++) get_scale_min_k4(j, x[i].scales, &scales[j], &mins[j]);
        int sumi = 0;
        for (int j = 0; j < QK_K / 16; ++j) sumi += y[i].bsums[j] * mins[j / 2];
        const int8_t *q8 = y[i].qs; a = aux8;
        for (int j = 0; j < QK_K / 32; ++j) {
            int32_t scale = scales[j];
            for (int g = 0; g < 4; g++) { for (int l = 0; l < 8; ++l) aux32[l] += scale * (q8[l] * a[l]); q8 += 8; a += 8; }
        }
        const float d = port_fp16_to_fp32(x[i].d) * y[i].d;
        for (int l = 0; l < 8; ++l) sums[l] += d * aux32[l];
        const float dmin = port_fp16_to_fp32(x[i].dmin) * y[i].d;
        sumf -= dmin * sumi;
    }
    for (int l = 0; l < 8; ++l) sumf += sums[l];
    return sumf;
}

/* ggml-quants.c:9523-9566 */
float port_vec_dot_q6_K_q8_K(int n, const void *vx, const void *vy) {
    const blk_q6_K *x = (const blk_q6_K *)vx; const blk_q8_K *y = (const blk_q8_K *)vy;
    float sums[8] = {0}; float sumf = 0;
    for (int i = 0; i < n / QK_K; ++i) {
        int32_t aux32[8] = {0};
        int8_t aux8[QK_K];
        const uint8_t *q4 = x[i].ql, *qh = x[i].qh; int8_t *a = aux8;
        for (int j = 0; j < QK_K; j += 128) {
            for (int l = 0; l < 32; ++l) {
                a[l +  0] = (int8_t)((q4[l +  0] & 0xF) | (((qh[l] >> 0) & 3) << 4)) - 32;
                a[l + 32] = (int8_t)((q4[l + 32] & 0xF) | (((qh[l] >> 2) & 3) << 4)) - 32;
                a[l + 64] = (int8_t)((q4[l +  0] >> 4) | (((qh[l] >> 4) & 3) << 4)) - 32;
                a[l + 96] = (int8_t)((q4[l + 32] >> 4) | (((qh[l] >> 6) & 3) << 4)) - 32;
            }
            a += 128; q4 += 64; qh += 32;
        }
        const int8_t *q8 = y[i].qs; a = aux8;
        for (int j = 0; j < QK_K / 16; ++j) {
            int scale = x[i].scales[j];
            for (int g = 0; g < 2; g++) { for (int l = 0; l < 8; ++l) aux32[l] += scale * (q8[l] * a[l]); q8 += 8; a += 8; }
        }
        const float d = port_fp16_to_fp32(x[i].d) * y[i].d;
        for (int l = 0; l < 8; ++l) sums[l] += d * aux32[l];
    }
    for (int l = 0; l < 8; ++l) sumf += sums[l];
    return sumf;
}

/* ggml-quants.c:5518-5860, scalar tail :5849-5857 */
float port_vec_dot_q8_0_q8_0(int n, const void *vx, const void *vy) {
    const blk_q8_0 *x = (const blk_q8_0 *)vx; const blk_q8_0 *y = (const blk_q8_0 *)vy;
    float sumf = 0;
    for (int ib = 0; ib < n / 32; ++ib) {
        int sumi = 0;
        for (int j = 0; j < 32; j++) sumi += x[ib].qs[j] * y[ib].qs[j];
        sumf += sumi * (port_fp16_to_fp32(x[ib].d) * port_fp16_to_fp32(y[ib].d));
    }
    return sumf;
}

/* ggml-quants.c:5144-5516, scalar tail :5489-5513 */
float port_vec_dot_q5_1_q8_1(int n, const void *vx, const void *vy) {
    const blk_q5_1 *x = (const blk_q5_1 *)vx; const blk_q8_1 *y = (const blk_q8_1 *)vy;
    float sumf = 0;
    for (int ib = 0; ib < n / 32; ++ib) {
        uint32_t qh; memcpy(&qh, x[ib].qh, 4);
        int sumi0 = 0, sumi1 = 0;
        for (int j = 0; j < 16; ++j) {
            const uint8_t xh_0 = ((qh >> (j + 0)) << 4) & 0x10;
            const uint8_t xh_1 = ((qh >> (j + 12))) & 0x10;
            const int32_t x0 = (x[ib].qs[j] & 0xF) | xh_0;
            const int32_t x1 = (x[ib].qs[j] >> 4) | xh_1;
            sumi0 += x0 * y[ib].qs[j];
            sumi1 += x1 * y[ib].qs[j + 16];
        }
        int sumi = sumi0 + sumi1;
        sumf += (port_fp16_to_fp32(x[ib].d) * port_fp16_to_fp32(y[ib].d)) * sumi
              + port_fp16_to_fp32(x[ib].m) * port_fp16_to_fp32(y[ib].s);
    }
    return sumf;
}

/* ggml-quants.c:3921-4500, scalar tail :4481-4496 */
float port_vec_dot_q4_0_q8_0(int n, const void *vx, const void *vy) {
    const blk_q4_0 *x = (const blk_q4_0 *)vx; const blk_q8_0 *y = (const blk_q8_0 *)vy;
    float sumf = 0;
    for (int ib = 0; ib < n / 32; ++ib) {
        int sumi0 = 0, sumi1 = 0;
        for (int j = 0; j < 16; ++j) {
            const int v0 = (x[ib].qs[j] & 0x0F) - 8;
            const int v1 = (x[ib].qs[j] >> 4) - 8;
            sumi0 += v0 * y[ib].qs[j];
            sumi1 += v1 * y[ib].qs[j + 16];
        }
        int sumi = sumi0 + sumi1;
        sumf += sumi * port_fp16_to_fp32(x[ib].d) * port_fp16_to_fp32(y[ib].d);
    }
    return sumf;
}

/* ggml-quants.c:4502-4787, scalar tail :4770-4783 */
float port_vec_dot_q4_1_q8_1(int n, const void *vx, const void *vy) {
    const blk_q4_1 *x = (const blk_q4_1 *)vx; const blk_q8_1 *y = (const blk_q8_1 *)vy;
    float sumf = 0;
    for (int ib = 0; ib < n / 32; ++ib) {
        int sumi0 = 0, sumi1 = 0;
        for (int j = 0; j < 16; ++j) {
            const int v0 = x[ib].qs[j] & 0x0F;
            const int v1 = x[ib].qs[j] >> 4;
            sumi0 += v0 * y[ib].qs[j];
            sumi1 += v1 * y[ib].qs[j + 16];
        }
        int sumi = sumi0 + sumi1;
        sumf += (port_fp16_to_fp32(x[ib].d) * port_fp16_to_fp32(y[ib].d)) * sumi
              + port_fp16_to_fp32(x[ib].m) * port_fp16_to_fp32(y[ib].s);
    }
    return sumf;
}

/* ggml-quants.c:4789-5142, scalar tail :5120-5138 */
float port_vec_dot_q5_0_q8_0(int n, const void *vx, const void *vy) {
    const blk_q5_0 *x = (const blk_q5_0 *)vx; const blk_q8_0 *y = (const blk_q8_0 *)vy;
    float sumf = 0;
    for (int ib = 0; ib < n / 32; ++ib) {
        uint32_t qh; memcpy(&qh, x[ib].qh, 4);
        int sumi0 = 0, sumi1 = 0;
        for (int j = 0; j < 16; ++j) {
            const uint8_t xh_0 = ((qh >> (j + 0)) << 4) & 0x10;
            const uint8_t xh_1 = ((qh >> (j + 12))) & 0x10;
            const int32_t x0 = ((x[ib].qs[j] & 0xF) | xh_0) - 16;
            const int32_t x1 = ((x[ib].qs[j] >> 4) | xh_1) - 16;
            sumi0 += x0 * y[ib].qs[j];
            sumi1 += x1 * y[ib].qs[j + 16];
        }
        int sumi = sumi0 + sumi1;
        sumf += (port_fp16_to_fp32(x[ib].d) * port_fp16_to_fp32(y[ib].d)) * sumi;
    }
    return sumf;
}

/* size in bytes of the activation row after conversion to the weight type's vec_dot_type
 * (type-traits table ggml.c:732-1100: Q4_K/Q5_K/Q6_K -> Q8_K, Q8_0/Q4_0/Q5_0 -> Q8_0, Q5_1/Q4_1 -> Q8_1, F16 -> F16) */
static int64_t act_row_size(int wtype, int64_t k) {
    switch (wtype) {
        case T_Q4_K: case T_Q5_K: case T_Q6_K: return k / 256 * (int64_t)sizeof(blk_q8_K);
        case T_Q8_0: case T_Q4_0: case T_Q5_0: return k / 32 * 34;
        case T_Q5_1: case T_Q4_1: return k / 32 * 36;
        case T_F16: return k * 2;
        default: return k * 4;
    }
}

static void act_quantize(int wtype, const float *x, void *q, int64_t k) {
    switch (wtype) {
        case T_Q4_K: case T_Q5_K: case T_Q6_K: port_quantize_row_q8_K(x, q, k); break;
        case T_Q8_0: case T_Q4_0: case T_Q5_0: port_quantize_row_q8_0(x, q, k); break;
        case T_Q5_1: case T_Q4_1: port_quantize_row_q8_1(x, q, k); break;
        case T_F16: for (int64_t i = 0; i < k; i++) ((uint16_t *)q)[i] = port_fp32_to_fp16(x[i]); break;
        default: memcpy(q, x, (size_t)k * 4);
    }
}

static float vec_dot(int wtype, int64_t k, const void *w, const void *q) {
    switch (wtype) {
        case T_Q4_K: return port_vec_dot_q4_K_q8_K((int)k, w, q);
        case T_Q5_K: return port_vec_dot_q5_K_q8_K((int)k, w, q);
        case T_Q6_K: return port_vec_dot_q6_K_q8_K((int)k, w, q);
        case T_Q8_0: return port_vec_dot_q8_0_q8_0((int)k, w, q);
        case T_Q5_1: return port_vec_dot_q5_1_q8_1((int)k, w, q);
        case T_Q4_0: return port_vec_dot_q4_0_q8_0((int)k, w, q);
        case T_Q4_1: return port_vec_dot_q4_1_q8_1((int)k, w, q);
        case T_Q5_0: return port_vec_dot_q5_0_q8_0((int)k, w, q);
        case T_F16: {  /* ggml_vec_dot_f16 ggml.c:1893-1930: f32 accumulation of f16*f16 */
            float s = 0; const uint16_t *a = (const uint16_t *)w, *b = (const uint16_t *)q;
            for (int64_t i = 0; i < k; i++) s += port_fp16_to_fp32(a[i]) * port_fp16_to_fp32(b[i]);
            return s;
        }
        default: { float s = 0; const float *a = (const float *)w, *b = (const float *)q;
                   for (int64_t i = 0; i < k; i++) s += a[i] * b[i]; return s; }
    }
}

/* ggml_compute_forward_mul_mat (ggml.c:12377-12600): dst[t][n] = W[n,:] . quant(x[t,:]) */
void port_mul_mat(int wtype, const void *W, int64_t N, int64_t K, const float *x, int64_t T, float *dst) {
    const int64_t rs = port_row_size(wtype, K);
    const int64_t as = act_row_size(wtype, K);
    void *q = malloc((size_t)as);
    for (int64_t t = 0; t < T; t++) {
        act_quantize(wtype, x + t * K, q, K);
        for (int64_t n = 0; n < N; n++) dst[t * N + n] = vec_dot(wtype, K, (const char *)W + n * rs, q);
    }
    free(q);
}

void port_quantize_act(int wtype, const float *x, void *q, int64_t k) { act_quantize(wtype, x, q, k); }
int64_t port_act_row_size(int wtype, int64_t k) { return act_row_size(wtype, k); }

/* ---------------- element-wise / normalisation ops ---------------- */
/* ggml.c:11950-11996: double-precision sum of squares, scale = 1/sqrtf(mean+eps) */
void port_rms_norm(const float *x, float *y, int64_t n, float eps) {
    double sum = 0.0;
    for (int64_t i = 0; i < n; i++) sum += (double)(x[i] * x[i]);
    const float mean = (float)(sum / n);
    const float scale = 1.0f / sqrtf(mean + eps);
    for (int64_t i = 0; i < n; i++) y[i] = x[i] * scale;
}

/* ggml.c:14087-14141 (yarn helpers) */
static float rope_yarn_ramp(const float low, const float high, const int i0) {
    const float y = (i0 / 2 - low) / fmaxf(0.001f, high - low);
    return 1 - fminf(1, fmaxf(0, y));
}
static float rope_yarn_corr_dim(int n_dims, int n_ctx_orig, float n_rot, float base) {
    return n_dims * logf(n_ctx_orig / (n_rot * 2 * (float)M_PI)) / (2 * logf(base));
}

/* ggml.c:14143-14266 ggml_compute_forward_rope_f32 for one token position.
 * x: [n_head][head_dim] contiguous; mode 0 = NORM (pairs i,i+1), mode 2 = NEOX (pairs i, i+n_dims/2). */
void port_rope(const float *x, float *y, int n_head, int head_dim, int n_dims, int mode, int32_t pos,
               float freq_base, float freq_scale, float ext_factor, float attn_factor,
               float beta_fast, float beta_slow, int n_ctx_orig, const float *freq_factors) {
    const float theta_scale = powf(freq_base, -2.0f / n_dims);
    float corr_dims[2];
    {
        float start = floorf(rope_yarn_corr_dim(n_dims, n_ctx_orig, beta_fast, freq_base));
        float end = ceilf(rope_yarn_corr_dim(n_dims, n_ctx_orig, beta_slow, freq_base));
        corr_dims[0] = fmaxf(0, start); corr_dims[1] = fminf(n_dims - 1, end);
    }
    float *cache = (float *)malloc(sizeof(float) * (size_t)head_dim);
    float theta = (float)pos;
    for (int i0 = 0; i0 < head_dim; i0 += 2) {
        const float ff = freq_factors ? freq_factors[i0 / 2] : 1.0f;
        float theta_extrap = theta / ff;
        float theta_interp = freq_scale * theta_extrap;
        float th = theta_interp, mscale = attn_factor;
        if (ext_factor != 0.0f) {
            float ramp_mix = rope_yarn_ramp(corr_dims[0], corr_dims[1], i0) * ext_factor;
            th = theta_interp * (1 - ramp_mix) + theta_extrap * ramp_mix;
            mscale *= 1.0f + 0.1f * logf(1.0f / freq_scale);
        }
        cache[i0] = cosf(th) * mscale; cache[i0 + 1] = sinf(th) * mscale;
        theta *= theta_scale;
    }
    for (int h = 0; h < n_head; h++) {
        const float *s = x + (size_t)h * head_dim; float *d = y + (size_t)h * head_dim;
        if (!(mode & 2)) {
            for (int i0 = 0; i0 < n_dims; i0 += 2) {
                const float c = cache[i0], sn = cache[i0 + 1], x0 = s[i0], x1 = s[i0 + 1];
                d[i0] = x0 * c - x1 * sn; d[i0 + 1] = x0 * sn + x1 * c;
            }
        } else {
            for (int i0 = 0; i0 < n_dims; i0 += 2) {
                const int ic = i0 / 2;
                const float c = cache[i0], sn = cache[i0 + 1], x0 = s[ic], x1 = s[ic + n_dims / 2];
                d[ic] = x0 * c - x1 * sn; d[ic + n_dims / 2] = x0 * sn + x1 * c;
            }
        }
        for (int i0 = n_dims; i0 < head_dim; i0++) d[i0] = s[i0];
    }
    free(cache);
}

/* ggml.c:13783-13880 soft_max_f32 (max_bias == 0): y = softmax(x*scale + mask) */
void port_soft_max(const float *x, const float *mask, float *y, int64_t n, float scale) {
    float mx = -INFINITY;
    for (int64_t i = 0; i < n; i++) { y[i] = x[i] * scale + (mask ? mask[i] : 0.0f); if (y[i] > mx) mx = y[i]; }
    double sum = 0.0;
    for (int64_t i = 0; i < n; i++) {
        if (y[i] == -INFINITY) { y[i] = 0.0f; } else { float v = expf(y[i] - mx); y[i] = v; sum += (double)v; }
    }
    const float inv = (float)(1.0 / sum);
    for (int64_t i = 0; i < n; i++) y[i] *= inv;
}

/* ggml.c:2560 ggml_silu_f32 */
static inline float silu_f32(float x) { return x / (1.0f + expf(-x)); }
void port_silu_mul(const float *gate, const float *up, float *y, int64_t n) {
    for (int64_t i = 0; i < n; i++) y[i] = silu_f32(gate[i]) * up[i];
}

/* Decode attention, FA-off numerics of the CPU backend (SURVEY §7.3 H1):
 *   kq[p]  = dot_f32( f16(K[p]), f16(q) )              ggml.c:12445-12473 (src1 -> vec_dot_type F16)
 *   p      = softmax(kq*scale + mask)   in f32          ggml.c:13783
 *   out[d] = dot_f32( V^T[d,:], f16(p) )                second mul_mat, src1 = probs -> f16
 * K cache: [n_ctx][n_head_kv*head_dim] f16; V cache: [n_ctx][n_head_kv*head_dim] f16 (token-major here;
 * the graph's transposed V layout holds the same values).  n_kv = number of valid cells (0..pos). */
void port_attention_decode(const float *q, const uint16_t *Kc, const uint16_t *Vc, float *out,
                           int n_head, int n_head_kv, int head_dim, int n_kv, float scale) {
    const int gqa = n_head / n_head_kv;
    const int64_t stride = (int64_t)n_head_kv * head_dim;
    float *kq = (float *)malloc(sizeof(float) * (size_t)n_kv);
    float *pr = (float *)malloc(sizeof(float) * (size_t)n_kv);
    uint16_t *q16 = (uint16_t *)malloc(2 * (size_t)head_dim);
    for (int h = 0; h < n_head; h++) {
        const int hk = h / gqa;
        for (int d = 0; d < head_dim; d++) q16[d] = port_fp32_to_fp16(q[(size_t)h * head_dim + d]);
        for (int p = 0; p < n_kv; p++) {
            const uint16_t *k = Kc + p * stride + (size_t)hk * head_dim;
            float s = 0;
            for (int d = 0; d < head_dim; d++) s += port_fp16_to_fp32(k[d]) * port_fp16_to_fp32(q16[d]);
            kq[p] = s;
        }
        port_soft_max(kq, NULL, pr, n_kv, scale);
        for (int d = 0; d < head_dim; d++) {
            float s = 0;
            for (int p = 0; p < n_kv; p++)
                s += port_fp16_to_fp32(Vc[p * stride + (size_t)hk * head_dim + d]) *
                     port_fp16_to_fp32(port_fp32_to_fp16(pr[p]));
            out[(size_t)h * head_dim + d] = s;
        }
    }
    free(kq); free(pr); free(q16);
}

/* ---------------- whole decode step (restates build_llama / build_qwen2, src/llama.cpp:11000-11216,
 * 12736-12916 with helpers :9673-9718, 9772-9929, 10032-10165; FA off) ---------------- */
typedef struct {
    int32_t n_layer, n_embd, n_head, n_head_kv, head_dim, n_ff, n_vocab, n_ctx;
    int32_t rope_mode;      /* 0 = NORM (llama), 2 = NEOX (qwen2) */
    int32_t n_ctx_orig;
    float rope_freq_base, rope_freq_scale, rms_eps;
} port_hparams;

typedef struct {
    int32_t type; int32_t _pad; const void *data;   /* raw GGUF blocks, row-major [N][K] */
} port_weight;

typedef struct {
    const float *attn_norm, *ffn_norm;
    port_weight wq, wk, wv, wo, gate, up, down;
    const float *bq, *bk, *bv;          /* qwen2 biases or NULL */
} port_layer;

typedef struct {
    port_hparams hp;
    port_weight tok_embd;               /* [n_vocab][n_embd] */
    const float *output_norm;
    port_weight output;                 /* [n_vocab][n_embd] */
    const port_layer *layers;
    const float *rope_freq_factors;     /* llama-3.1 or NULL */
    uint16_t *k_cache, *v_cache;        /* [n_layer][n_ctx][n_head_kv*head_dim] f16, caller-owned */
} port_model;

/* one token at position pos; writes n_vocab logits; hidden_out (optional) gets the last layer output */
void port_llama_decode(const port_model *m, int32_t token, int32_t pos, float *logits, float *hidden_out) {
    const port_hparams *hp = &m->hp;
    const int E = hp->n_embd, H = hp->n_head, HK = hp->n_head_kv, D = hp->head_dim, F = hp->n_ff;
    const int EK = HK * D;
    float *x = (float *)malloc(sizeof(float) * (size_t)E), *cur = (float *)malloc(sizeof(float) * (size_t)E);
    float *qv = (float *)malloc(sizeof(float) * (size_t)H * D), *kv = (float *)malloc(sizeof(float) * (size_t)EK);
    float *vv = (float *)malloc(sizeof(float) * (size_t)EK), *att = (float *)malloc(sizeof(float) * (size_t)H * D);
    float *tmp = (float *)malloc(sizeof(float) * (size_t)(E > H * D ? E : H * D));
    float *g = (float *)malloc(sizeof(float) * (size_t)F), *u = (float *)malloc(sizeof(float) * (size_t)F);
    /* get_rows on token_embd (ggml.c get_rows_q: dequantize_row of one row) */
    port_dequantize_row(m->tok_embd.type, (const char *)m->tok_embd.data + (int64_t)token * port_row_size(m->tok_embd.type, E), x, E);
    const float kq_scale = 1.0f / sqrtf((float)D);
    for (int il = 0; il < hp->n_layer; il++) {
        const port_layer *L = &m->layers[il];
        uint16_t *Kc = m->k_cache + (size_t)il * hp->n_ctx * EK, *Vc = m->v_cache + (size_t)il * hp->n_ctx * EK;
        port_rms_norm(x, cur, E, hp->rms_eps);
        for (int i = 0; i < E; i++) cur[i] *= L->attn_norm[i];
        port_mul_mat(L->wq.type, L->wq.data, (int64_t)H * D, E, cur, 1, qv);
        port_mul_mat(L->wk.type, L->wk.data, EK, E, cur, 1, kv);
        port_mul_mat(L->wv.type, L->wv.data, EK, E, cur, 1, vv);
        if (L->bq) for (int i = 0; i < H * D; i++) qv[i] += L->bq[i];
        if (L->bk) for (int i = 0; i < EK; i++) kv[i] += L->bk[i];
        if (L->bv) for (int i = 0; i < EK; i++) vv[i] += L->bv[i];
        port_rope(qv, qv, H, D, D, hp->rope_mode, pos, hp->rope_freq_base, hp->rope_freq_scale, 0.0f, 1.0f, 32.0f, 1.0f, hp->n_ctx_orig, m->rope_freq_factors);
        port_rope(kv, kv, HK, D, D, hp->rope_mode, pos, hp->rope_freq_base, hp->rope_freq_scale, 0.0f, 1.0f, 32.0f, 1.0f, hp->n_ctx_orig, m->rope_freq_factors);
        for (int i = 0; i < EK; i++) { Kc[(size_t)pos * EK + i] = port_fp32_to_fp16(kv[i]); Vc[(size_t)pos * EK + i] = port_fp32_to_fp16(vv[i]); }
        port_attention_decode(qv, Kc, Vc, att, H, HK, D, pos + 1, kq_scale);
        port_mul_mat(L->wo.type, L->wo.data, E, (int64_t)H * D, att, 1, tmp);
        for (int i = 0; i < E; i++) x[i] = tmp[i] + x[i];            /* ffn_inp = cur + inpSA */
        port_rms_norm(x, cur, E, hp->rms_eps);
        for (int i = 0; i < E; i++) cur[i] *= L->ffn_norm[i];
        port_mul_mat(L->up.type, L->up.data, F, E, cur, 1, u);
        port_mul_mat(L->gate.type, L->gate.data, F, E, cur, 1, g);
        port_silu_mul(g, u, g, F);
        port_mul_mat(L->down.type, L->down.data, E, F, g, 1, tmp);
        for (int i = 0; i < E; i++) x[i] = tmp[i] + x[i];
    }
    if (hidden_out) memcpy(hidden_out, x, sizeof(float) * (size_t)E);
    if (logits) {
        port_rms_norm(x, cur, E, hp->rms_eps);
        for (int i = 0; i < E; i++) cur[i] *= m->output_norm[i];
        port_mul_mat(m->output.type, m->output.data, hp->n_vocab, E, cur, 1, logits);
    }
    free(x); free(cur); free(qv); free(kv); free(vv); free(att); free(tmp); free(g); free(u);
}
