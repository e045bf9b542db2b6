// exb_math.h -- host/device math shared by the CPU core and the sm_90a kernels.
//
// One definition of every sparse optimizer and every initializer so that the CPU
// engine (oracle, gloo path) and the CUDA engine compute the same thing.
//
// Behavioural parity targets (reference, read-only):
//   optimizers   openembedding/variable/EmbeddingOptimizer.h:49-390
//   initializers openembedding/variable/EmbeddingInitializer.h:20-93
// Design differences (deliberate, GPU-first):
//   * row update is expressed per element (+ a per-row scalar prologue) so a lane
//     group of a warp can update one row cooperatively with float4 accesses;
//   * initializers are counter-based (Philox4x32-10 keyed by (seed, variable, row))
//     instead of a stateful std::default_random_engine: any GPU can compute the
//     initial value of any row without communication or locks, which is what makes
//     the one-sided peer "pull" of never-touched hash rows possible.
#pragma once
#include <stdint.h>
#include <math.h>

#if defined(__CUDACC__)
#define EXB_HD __host__ __device__ __forceinline__
#else
#define EXB_HD inline
#endif

namespace exb {

// ---------------------------------------------------------------- optimizers
enum OptKind : int {
    OPT_DEFAULT = 0,  // stateless SGD, lr default 0
    OPT_ADADELTA = 1,
    OPT_ADAGRAD = 2,
    OPT_ADAM = 3,
    OPT_ADAMAX = 4,
    OPT_FTRL = 5,
    OPT_RMSPROP = 6,
    OPT_SGD = 7,
    OPT_TEST = 8,
    OPT_NUM_KINDS = 9
};

// Hyper-parameters, meaning of p[] per kind (kept as double, cast to T at use):
//  default : p0 lr
//  adadelta: p0 lr, p1 rho, p2 eps
//  adagrad : p0 lr, p1 initial_accumulator_value, p2 eps
//  adam    : p0 lr, p1 beta_1, p2 beta_2, p3 eps
//  adamax  : p0 lr, p1 beta_1, p2 beta_2, p3 eps
//  ftrl    : p0 lr, p1 initial_accumulator_value, p2 l1, p3 l2, p4 l2_shrinkage,
//            p5 learning_rate_power, p6 beta
//  rmsprop : p0 lr, p1 rho, p2 momentum, p3 eps
//  sgd     : p0 lr, p1 momentum, p2 nesterov(0/1)
//  test    : p0 lr, p1 flip, p2 init
struct OptParams {
    int kind;
    int _pad;
    double p[8];
};

// number of per-element state slots and trailing per-row scalars
EXB_HD int opt_num_slots(int kind) {
    switch (kind) {
        case OPT_ADADELTA: return 2;
        case OPT_ADAGRAD: return 1;
        case OPT_ADAM: return 2;
        case OPT_ADAMAX: return 2;
        case OPT_FTRL: return 2;
        case OPT_RMSPROP: return 2;
        case OPT_SGD: return 1;
        default: return 0;
    }
}
EXB_HD int opt_num_scalars(int kind) {
    switch (kind) {
        case OPT_ADAM: return 2;
        case OPT_ADAMAX: return 1;
        case OPT_TEST: return 2;
        default: return 0;
    }
}
EXB_HD int opt_state_dim(int kind, int dim) {
    return opt_num_slots(kind) * dim + opt_num_scalars(kind);
}

// initial value of element-wise slot `slot`
template <class T>
EXB_HD T opt_slot_init(const OptParams& P, int slot) {
    if ((P.kind == OPT_ADAGRAD || P.kind == OPT_FTRL) && slot == 0) return (T)P.p[1];
    return (T)0;
}
// initial value of trailing scalar `i`
template <class T>
EXB_HD T opt_scalar_init(const OptParams& P, int i) {
    if (P.kind == OPT_ADAM || P.kind == OPT_ADAMAX) return (T)1;
    if (P.kind == OPT_TEST) return i == 0 ? (T)P.p[2] : (T)0;
    return (T)0;
}

template <class T>
struct RowCtx {  // per-row values computed once by the prologue
    T a, b;
};

// fp32 on the device: approximate sqrt / divide (sqrt.approx: 1 ulp, div.approx: 2 ulp). The
// IEEE sequences cost ~15 instructions each with a slow-path branch and made the apply phase
// of the push kernel issue bound (73 instructions per element for Adagrad).
#if defined(__CUDA_ARCH__)
EXB_HD float exb_sqrt(float x) { float r; asm("sqrt.approx.f32 %0, %1;" : "=f"(r) : "f"(x)); return r; }
EXB_HD float exb_div(float a, float b) { return __fdividef(a, b); }
#else
EXB_HD float exb_sqrt(float x) { return sqrtf(x); }
EXB_HD float exb_div(float a, float b) { return a / b; }
#endif
EXB_HD double exb_sqrt(double x) { return sqrt(x); }
EXB_HD double exb_div(double a, double b) { return a / b; }
EXB_HD float exb_pow(float x, float y) { return powf(x, y); }
EXB_HD double exb_pow(double x, double y) { return pow(x, y); }
EXB_HD float exb_abs(float x) { return fabsf(x); }
EXB_HD double exb_abs(double x) { return fabs(x); }
template <class T> EXB_HD T exb_max(T a, T b) { return a > b ? a : b; }
template <class T> EXB_HD T exb_min(T a, T b) { return a < b ? a : b; }

// Per-row prologue. `scalars` points at the trailing scalars of the row state (may be
// null when the optimizer has none). Updates them in place (caller guarantees a single
// writer per row) and returns what the element update needs.
template <class T>
EXB_HD RowCtx<T> opt_row_prologue(const OptParams& P, T* scalars, uint64_t count) {
    RowCtx<T> rc;
    rc.a = (T)0;
    rc.b = (T)0;
    switch (P.kind) {
        case OPT_ADAM: {
            T b1t = scalars[0] * (T)P.p[1];
            T b2t = scalars[1] * (T)P.p[2];
            scalars[0] = b1t;
            scalars[1] = b2t;
            rc.a = (T)P.p[0] * exb_sqrt((T)1 - b2t) / ((T)1 - b1t);  // lr_t
            break;
        }
        case OPT_ADAMAX: {
            T b1t = scalars[0] * (T)P.p[1];
            scalars[0] = b1t;
            rc.a = (T)P.p[0] / ((T)1 - b1t);  // lr_t
            break;
        }
        case OPT_TEST: {
            T s = (T)P.p[1] - scalars[0];
            scalars[0] = s;
            rc.a = s;
            rc.b = (T)(count ? count : 1);
            break;
        }
        default: break;
    }
    return rc;
}

// Same as above but without side effects: used when a lane group evaluates the
// prologue redundantly and only one lane commits the scalars.
template <class T>
EXB_HD RowCtx<T> opt_row_prologue_pure(const OptParams& P, const T* scalars, uint64_t count,
                                       T* new_scalars /* [2] */) {
    T tmp[2] = {(T)0, (T)0};
    int ns = opt_num_scalars(P.kind);
    for (int i = 0; i < ns; ++i) tmp[i] = scalars[i];
    RowCtx<T> rc = opt_row_prologue<T>(P, tmp, count);
    new_scalars[0] = tmp[0];
    new_scalars[1] = tmp[1];
    return rc;
}

// Element update: w, s0, s1 are updated in place; g is the summed gradient.
template <class T>
EXB_HD void opt_elem(const OptParams& P, const RowCtx<T>& rc, T& w, T& s0, T& s1, T g) {
    switch (P.kind) {
        case OPT_DEFAULT: {
            T lr = (T)P.p[0];
            if (lr != (T)0) w -= lr * g;
            break;
        }
        case OPT_ADADELTA: {
            T lr = (T)P.p[0], rho = (T)P.p[1], eps = (T)P.p[2];
            s0 = s0 * rho + g * g * ((T)1 - rho);
            T upd = exb_div(g * exb_sqrt(s1 + eps), exb_sqrt(s0 + eps));
            s1 = s1 * rho + upd * upd * ((T)1 - rho);
            w -= lr * upd;
            break;
        }
        case OPT_ADAGRAD: {
            T lr = (T)P.p[0], eps = (T)P.p[2];
            s0 += g * g;
            w -= exb_div(lr * g, exb_sqrt(s0) + eps);
            break;
        }
        case OPT_ADAM: {
            T b1 = (T)P.p[1], b2 = (T)P.p[2], eps = (T)P.p[3];
            s0 = s0 * b1 + g * ((T)1 - b1);
            s1 = s1 * b2 + g * g * ((T)1 - b2);
            w -= exb_div(rc.a * s0, exb_sqrt(s1) + eps);
            break;
        }
        case OPT_ADAMAX: {
            T b1 = (T)P.p[1], b2 = (T)P.p[2], eps = (T)P.p[3];
            s0 = s0 * b1 + g * ((T)1 - b1);
            s1 = exb_max(exb_abs(g), s1 * b2);
            w -= exb_div(rc.a * s0, s1 + eps);
            break;
        }
        case OPT_FTRL: {
            T lr = (T)P.p[0], l1 = (T)P.p[2], l2 = (T)P.p[3], l2s = (T)P.p[4];
            T lrp = (T)P.p[5], beta = (T)P.p[6];
            T adj_l2 = l2 + beta / lr / (T)2;
            T gg = g + (T)2 * l2s * w;
            T accum_new = s0 + g * g;
            T pa, pn;
            if (lrp == (T)-0.5) {
                pa = exb_sqrt(s0);
                pn = exb_sqrt(accum_new);
            } else {
                pa = exb_pow(s0, -lrp);
                pn = exb_pow(accum_new, -lrp);
            }
            T sigma = (pn - pa) / lr;
            s1 += gg - sigma * w;  // linear
            s0 = accum_new;
            T quadratic = pn / lr + (T)2 * adj_l2;
            T l1_adj = exb_max(exb_min(s1, l1), -l1);
            w = exb_div(l1_adj - s1, quadratic);
            break;
        }
        case OPT_RMSPROP: {
            T lr = (T)P.p[0], rho = (T)P.p[1], mom = (T)P.p[2], eps = (T)P.p[3];
            s0 = s0 * rho + g * g * ((T)1 - rho);
            s1 = s1 * mom + exb_div(lr * g, exb_sqrt(s0 + eps));
            w -= s1;
            break;
        }
        case OPT_SGD: {
            T lr = (T)P.p[0], mom = (T)P.p[1];
            s0 = s0 * mom + lr * g;
            if (P.p[2] != 0.0) w -= s0 * mom + lr * g;
            else w -= s0;
            break;
        }
        case OPT_TEST: {
            w += (T)P.p[0] * g / rc.b + rc.a;
            break;
        }
        default: break;
    }
}

// Whole-row update on one thread (CPU engine and tail paths). state layout:
// [slot0[dim] | slot1[dim] | scalars]
template <class T>
EXB_HD void opt_update_row(const OptParams& P, T* w, T* state, int dim, uint64_t count,
                           const T* g) {
    int nslots = opt_num_slots(P.kind);
    T* scalars = state + (size_t)nslots * dim;
    RowCtx<T> rc = opt_row_prologue<T>(P, opt_num_scalars(P.kind) ? scalars : (T*)0, count);
    for (int i = 0; i < dim; ++i) {
        T d0 = (T)0, d1 = (T)0;
        T& s0 = nslots > 0 ? state[i] : d0;
        T& s1 = nslots > 1 ? state[dim + i] : d1;
        opt_elem<T>(P, rc, w[i], s0, s1, g[i]);
    }
}

template <class T>
EXB_HD void opt_init_state(const OptParams& P, T* state, int dim) {
    int nslots = opt_num_slots(P.kind);
    for (int s = 0; s < nslots; ++s)
        for (int i = 0; i < dim; ++i) state[(size_t)s * dim + i] = opt_slot_init<T>(P, s);
    int ns = opt_num_scalars(P.kind);
    for (int i = 0; i < ns; ++i) state[(size_t)nslots * dim + i] = opt_scalar_init<T>(P, i);
}

// -------------------------------------------------------------- initializers
enum InitKind : int { INIT_CONSTANT = 0, INIT_UNIFORM = 1, INIT_NORMAL = 2 };

// constant: p0 value | uniform: p0 minval, p1 maxval | normal: p0 mean, p1 stddev, p2 truncated
struct InitParams {
    int kind;
    int _pad;
    double p[3];
    uint64_t seed;  // (user seed, variable id) mixed by the host
};

struct Philox4 {
    uint32_t v[4];
};

EXB_HD uint32_t exb_mulhi32(uint32_t a, uint32_t b) {
#if defined(__CUDA_ARCH__)
    return __umulhi(a, b);
#else
    return (uint32_t)(((uint64_t)a * (uint64_t)b) >> 32);
#endif
}

// Philox4x32-10 (Salmon et al.), counter = (c0..c3), key = (k0,k1)
EXB_HD Philox4 philox4x32_10(uint32_t c0, uint32_t c1, uint32_t c2, uint32_t c3, uint32_t k0,
                             uint32_t k1) {
    const uint32_t M0 = 0xD2511F53u, M1 = 0xCD9E8D57u, W0 = 0x9E3779B9u, W1 = 0xBB67AE85u;
#if defined(__CUDA_ARCH__)
#pragma unroll
#endif
    for (int r = 0; r < 10; ++r) {
        uint32_t hi0 = exb_mulhi32(M0, c0), lo0 = M0 * c0;
        uint32_t hi1 = exb_mulhi32(M1, c2), lo1 = M1 * c2;
        uint32_t n0 = hi1 ^ c1 ^ k0;
        uint32_t n1 = lo1;
        uint32_t n2 = hi0 ^ c3 ^ k1;
        uint32_t n3 = lo0;
        c0 = n0; c1 = n1; c2 = n2; c3 = n3;
        k0 += W0; k1 += W1;
    }
    Philox4 o;
    o.v[0] = c0; o.v[1] = c1; o.v[2] = c2; o.v[3] = c3;
    return o;
}

EXB_HD float exb_u01(uint32_t x, float) {  // (0,1]-free uniform in [0,1)
    return (float)(x >> 8) * (1.0f / 16777216.0f);
}
EXB_HD double exb_u01(uint32_t hi, uint32_t lo, double) {
    uint64_t v = (((uint64_t)hi << 32) | lo) >> 11;
    return (double)v * (1.0 / 9007199254740992.0);
}

EXB_HD float exb_fma(float a, float b, float c) {
#if defined(__CUDA_ARCH__)
    return __fmaf_rn(a, b, c);
#else
    return fmaf(a, b, c);
#endif
}
EXB_HD double exb_fma(double a, double b, double c) {
#if defined(__CUDA_ARCH__)
    return __fma_rn(a, b, c);
#else
    return fma(a, b, c);
#endif
}

// Initial value of element `col` of row `row` (global id / hash key) -- pure function.
// Elements are generated in blocks of 4 (one Philox call per 4 fp32 elements, per 2 fp64).
template <class T>
struct InitGen;

template <>
struct InitGen<float> {
    // fills out[0..3] = elements 4*blk .. 4*blk+3 of the row
    static EXB_HD void block4(const InitParams& I, uint64_t row, uint32_t blk, float* out) {
        if (I.kind == INIT_CONSTANT) {
            out[0] = out[1] = out[2] = out[3] = (float)I.p[0];
            return;
        }
        uint32_t k0 = (uint32_t)I.seed, k1 = (uint32_t)(I.seed >> 32);
        uint32_t r0 = (uint32_t)row, r1 = (uint32_t)(row >> 32);
        if (I.kind == INIT_UNIFORM) {
            Philox4 r = philox4x32_10(r0, r1, blk, 0u, k0, k1);
            float lo = (float)I.p[0], range = (float)(I.p[1] - I.p[0]);
            for (int i = 0; i < 4; ++i) out[i] = exb_fma(exb_u01(r.v[i], 0.f), range, lo);
            return;
        }
        // normal (Box-Muller, 2 normals per 2 uniforms); truncated: resample while
        // (x-mean)/stddev > truncated, one-sided like the reference
        // (EmbeddingInitializer.h:76-81), bounded to 8 attempts then clamped.
        float mean = (float)I.p[0], sd = (float)I.p[1], tr = (float)I.p[2];
        float z[4];
        Philox4 r = philox4x32_10(r0, r1, blk, 0u, k0, k1);
        for (int h = 0; h < 2; ++h) {
            float u1 = 1.0f - exb_u01(r.v[2 * h], 0.f);  // (0,1]
            float u2 = exb_u01(r.v[2 * h + 1], 0.f);
            float rad = sqrtf(-2.0f * logf(u1));
            float ang = 6.283185307179586f * u2;
            z[2 * h] = rad * cosf(ang);
            z[2 * h + 1] = rad * sinf(ang);
        }
        if (tr > 0.1f) {
            for (int i = 0; i < 4; ++i) {
                uint32_t attempt = 1;
                while (z[i] > tr && attempt <= 8) {
                    Philox4 q = philox4x32_10(r0, r1, blk, attempt * 4u + (uint32_t)i, k0, k1);
                    float u1 = 1.0f - exb_u01(q.v[0], 0.f), u2 = exb_u01(q.v[1], 0.f);
                    z[i] = sqrtf(-2.0f * logf(u1)) * cosf(6.283185307179586f * u2);
                    ++attempt;
                }
                if (z[i] > tr) z[i] = tr;
            }
        }
        for (int i = 0; i < 4; ++i) out[i] = exb_fma(z[i], sd, mean);
    }
};

template <>
struct InitGen<double> {
    static EXB_HD void block4(const InitParams& I, uint64_t row, uint32_t blk, double* out) {
        if (I.kind == INIT_CONSTANT) {
            out[0] = out[1] = out[2] = out[3] = I.p[0];
            return;
        }
        uint32_t k0 = (uint32_t)I.seed, k1 = (uint32_t)(I.seed >> 32);
        uint32_t r0 = (uint32_t)row, r1 = (uint32_t)(row >> 32);
        // two Philox calls give 8 words = 4 doubles worth of uniforms
        Philox4 a = philox4x32_10(r0, r1, blk, 0x80000000u, k0, k1);
        Philox4 b = philox4x32_10(r0, r1, blk, 0x80000001u, k0, k1);
        double u[4] = {exb_u01(a.v[0], a.v[1], 0.0), exb_u01(a.v[2], a.v[3], 0.0),
                       exb_u01(b.v[0], b.v[1], 0.0), exb_u01(b.v[2], b.v[3], 0.0)};
        if (I.kind == INIT_UNIFORM) {
            for (int i = 0; i < 4; ++i) out[i] = exb_fma(u[i], I.p[1] - I.p[0], I.p[0]);
            return;
        }
        double mean = I.p[0], sd = I.p[1], tr = I.p[2];
        double z[4];
        for (int h = 0; h < 2; ++h) {
            double u1 = 1.0 - u[2 * h], u2 = u[2 * h + 1];
            double rad = sqrt(-2.0 * log(u1)), ang = 6.283185307179586 * u2;
            z[2 * h] = rad * cos(ang);
            z[2 * h + 1] = rad * sin(ang);
        }
        if (tr > 0.1) {
            for (int i = 0; i < 4; ++i) {
                uint32_t attempt = 1;
                while (z[i] > tr && attempt <= 8) {
                    Philox4 q = philox4x32_10(r0, r1, blk, 0x80000002u + attempt * 4u + (uint32_t)i,
                                              k0, k1);
                    double u1 = 1.0 - exb_u01(q.v[0], q.v[1], 0.0);
                    double u2 = exb_u01(q.v[2], q.v[3], 0.0);
                    z[i] = sqrt(-2.0 * log(u1)) * cos(6.283185307179586 * u2);
                    ++attempt;
                }
                if (z[i] > tr) z[i] = tr;
            }
        }
        for (int i = 0; i < 4; ++i) out[i] = exb_fma(z[i], sd, mean);
    }
};

template <class T>
EXB_HD void init_row(const InitParams& I, uint64_t row, T* w, int dim) {
    for (int blk = 0; blk * 4 < dim; ++blk) {
        T tmp[4];
        InitGen<T>::block4(I, row, (uint32_t)blk, tmp);
        for (int i = 0; i < 4 && blk * 4 + i < dim; ++i) w[blk * 4 + i] = tmp[i];
    }
}

// 64-bit mix used for hash-table slot selection (splitmix64 finaliser)
EXB_HD uint64_t exb_hash64(uint64_t x) {
    x ^= x >> 30; x *= 0xbf58476d1ce4e5b9ull;
    x ^= x >> 27; x *= 0x94d049bb133111ebull;
    x ^= x >> 31;
    return x;
}

}  // namespace exb
