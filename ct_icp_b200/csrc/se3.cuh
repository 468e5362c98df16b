// se3.cuh — fp64 SE3 / quaternion algebra shared by host orchestration and sm_90a kernels.
//
// Restates the arithmetic the reference gets from Eigen + slam::TSE3/TPose
// (include/SlamCore/types.h:100-139, 192-219, 313-366, 434-470): quaternion product, q·v, slerp (not renormalised),
// Quaternion(Matrix3), toRotationMatrix, pose interpolation. Everything is fp64: world coordinates reach km and the
// parity budget is 1e-4 m (SURVEY §7 "Precision").
#pragma once
#include <cmath>
#include <cstdint>

#ifdef __CUDACC__
#define CT_HD __host__ __device__ __forceinline__
#else
#define CT_HD inline
#endif

namespace cticp {

struct V3 {
    double x, y, z;
};
CT_HD V3 mk(double x, double y, double z) { return V3{x, y, z}; }
CT_HD V3 operator+(V3 a, V3 b) { return {a.x + b.x, a.y + b.y, a.z + b.z}; }
CT_HD V3 operator-(V3 a, V3 b) { return {a.x - b.x, a.y - b.y, a.z - b.z}; }
CT_HD V3 operator*(double s, V3 a) { return {s * a.x, s * a.y, s * a.z}; }
CT_HD double dot(V3 a, V3 b) { return a.x * b.x + a.y * b.y + a.z * b.z; }
CT_HD V3 cross(V3 a, V3 b) { return {a.y * b.z - a.z * b.y, a.z * b.x - a.x * b.z, a.x * b.y - a.y * b.x}; }
CT_HD double norm(V3 a) { return sqrt(dot(a, a)); }

struct Q4 {   // (x, y, z, w) like Eigen::Quaterniond::coeffs()
    double x, y, z, w;
};
CT_HD Q4 qmul(Q4 a, Q4 b) {
    return {a.w * b.x + a.x * b.w + a.y * b.z - a.z * b.y, a.w * b.y + a.y * b.w + a.z * b.x - a.x * b.z,
            a.w * b.z + a.z * b.w + a.x * b.y - a.y * b.x, a.w * b.w - a.x * b.x - a.y * b.y - a.z * b.z};
}
CT_HD double qdot(Q4 a, Q4 b) { return a.x * b.x + a.y * b.y + a.z * b.z + a.w * b.w; }
CT_HD Q4 qnormalized(Q4 q) {
    double n = sqrt(qdot(q, q));
    return {q.x / n, q.y / n, q.z / n, q.w / n};
}
CT_HD Q4 qinverse(Q4 q) {   // Eigen inverse(): conjugate / squaredNorm
    double n2 = qdot(q, q);
    if (n2 > 0) return {-q.x / n2, -q.y / n2, -q.z / n2, q.w / n2};
    return {0, 0, 0, 0};
}
// Eigen _transformVector: uv = 2 (q.vec × v); v + w uv + q.vec × uv
CT_HD V3 qrot(Q4 q, V3 v) {
    V3 qv = {q.x, q.y, q.z};
    V3 uv = cross(qv, v);
    uv = uv + uv;
    return v + q.w * uv + cross(qv, uv);
}
// Eigen slerp (types.h:363): result NOT renormalised
CT_HD Q4 qslerp(Q4 a, Q4 b, double t) {
    const double one = 1.0 - 2.220446049250313e-16;
    double d = qdot(a, b);
    double ad = fabs(d);
    double s0, s1;
    if (ad >= one) {
        s0 = 1.0 - t;
        s1 = t;
    } else {
        double theta = acos(ad);
        double st = sin(theta);
        s0 = sin((1.0 - t) * theta) / st;
        s1 = sin(t * theta) / st;
    }
    if (d < 0) s1 = -s1;
    return {s0 * a.x + s1 * b.x, s0 * a.y + s1 * b.y, s0 * a.z + s1 * b.z, s0 * a.w + s1 * b.w};
}
// The angle between the two poses of a frame is the same for every point of the frame: acos / sin(theta) are
// evaluated once per ICP iteration (SlerpConsts) and each point only pays for sin((1-t) theta) and sin(t theta).
struct SlerpConsts {
    double theta, inv_sin;
    int linear;      // |d| >= 1 - eps  → plain lerp branch of Eigen's slerp
    int negate;      // d < 0           → scale1 = -scale1
};
CT_HD SlerpConsts slerp_consts(Q4 a, Q4 b) {
    const double one = 1.0 - 2.220446049250313e-16;
    SlerpConsts c;
    const double d = qdot(a, b);
    const double ad = fabs(d);
    c.linear = ad >= one;
    c.negate = d < 0;
    c.theta = c.linear ? 0.0 : acos(ad);
    // sin(acos(ad)) = sqrt((1 - ad)(1 + ad)): one sqrt instead of a second transcendental, and more accurate near 1
    c.inv_sin = c.linear ? 0.0 : 1.0 / sqrt((1.0 - ad) * (1.0 + ad));
    return c;
}
// sin(x) for |x| <= 0.5 by its Taylor series up to x^17 (next term 0.5^19 / 19! = 1.6e-23: below half an ulp): ten
// dependent FMAs instead of libm's argument reduction. The slerp angle of one sweep is a few degrees at most.
CT_HD double sin_upto_half(double x) {
    const double x2 = x * x;
    double p = 2.8114572543455206e-15;          //  1/17!
    p = p * x2 - 7.647163731819816e-13;         // -1/15!
    p = p * x2 + 1.6059043836821613e-10;        //  1/13!
    p = p * x2 - 2.505210838544172e-8;          // -1/11!
    p = p * x2 + 2.7557319223985893e-6;         //  1/9!
    p = p * x2 - 1.984126984126984e-4;          // -1/7!
    p = p * x2 + 8.333333333333333e-3;          //  1/5!
    p = p * x2 - 0.16666666666666666;           // -1/3!
    return x + x * (x2 * p);
}
// cos(x) for |x| <= 0.5, Taylor up to x^18 (next term 0.5^20 / 20! = 3.9e-25)
CT_HD double cos_upto_half(double x) {
    const double x2 = x * x;
    double p = 1.5619206968586226e-16;          //  1/18!
    p = p * x2 - 4.779477332387385e-14;         // -1/16!
    p = p * x2 + 1.1470745597729725e-11;        //  1/14!
    p = p * x2 - 2.08767569878681e-9;           // -1/12!
    p = p * x2 + 2.755731922398589e-7;          //  1/10!
    p = p * x2 - 2.48015873015873e-5;           // -1/8!
    p = p * x2 + 1.388888888888889e-3;          //  1/6!
    p = p * x2 - 4.1666666666666664e-2;         // -1/4!
    p = p * x2 + 0.5;                           //  1/2!
    return 1.0 - x2 * p;
}
CT_HD Q4 qslerp_c(Q4 a, Q4 b, double t, const SlerpConsts &c) {
    double s0, s1;
    if (c.linear) {
        s0 = 1.0 - t;
        s1 = t;
    } else if (c.theta <= 0.5) {   // t in [0, 1] for every point of the sweep
        s0 = sin_upto_half((1.0 - t) * c.theta) * c.inv_sin;
        s1 = sin_upto_half(t * c.theta) * c.inv_sin;
    } else {
        s0 = sin((1.0 - t) * c.theta) * c.inv_sin;
        s1 = sin(t * c.theta) * c.inv_sin;
    }
    if (c.negate) s1 = -s1;
    return {s0 * a.x + s1 * b.x, s0 * a.y + s1 * b.y, s0 * a.z + s1 * b.z, s0 * a.w + s1 * b.w};
}
struct M3 {
    double m[3][3];
};
CT_HD M3 qtoR(Q4 q) {
    M3 r;
    const double tx = 2 * q.x, ty = 2 * q.y, tz = 2 * q.z;
    const double twx = tx * q.w, twy = ty * q.w, twz = tz * q.w;
    const double txx = tx * q.x, txy = ty * q.x, txz = tz * q.x;
    const double tyy = ty * q.y, tyz = tz * q.y, tzz = tz * q.z;
    r.m[0][0] = 1 - (tyy + tzz); r.m[0][1] = txy - twz; r.m[0][2] = txz + twy;
    r.m[1][0] = txy + twz; r.m[1][1] = 1 - (txx + tzz); r.m[1][2] = tyz - twx;
    r.m[2][0] = txz - twy; r.m[2][1] = tyz + twx; r.m[2][2] = 1 - (txx + tyy);
    return r;
}
CT_HD M3 mmul(const M3 &a, const M3 &b) {
    M3 r;
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) r.m[i][j] = a.m[i][0] * b.m[0][j] + a.m[i][1] * b.m[1][j] + a.m[i][2] * b.m[2][j];
    return r;
}
// Eigen Quaternion(Matrix3) (trace-based), used by the GN pose update (src/ct_icp/ct_icp.cpp:950-954)
CT_HD Q4 qfromR(const M3 &R) {
    Q4 q;
    double t = R.m[0][0] + R.m[1][1] + R.m[2][2];
    if (t > 0) {
        t = sqrt(t + 1.0);
        q.w = 0.5 * t;
        t = 0.5 / t;
        q.x = (R.m[2][1] - R.m[1][2]) * t;
        q.y = (R.m[0][2] - R.m[2][0]) * t;
        q.z = (R.m[1][0] - R.m[0][1]) * t;
    } else {
        int i = 0;
        if (R.m[1][1] > R.m[0][0]) i = 1;
        if (R.m[2][2] > R.m[i][i]) i = 2;
        int j = (i + 1) % 3, k = (j + 1) % 3;
        t = sqrt(R.m[i][i] - R.m[j][j] - R.m[k][k] + 1.0);
        double c[3];
        c[i] = 0.5 * t;
        t = 0.5 / t;
        q.w = (R.m[k][j] - R.m[j][k]) * t;
        c[j] = (R.m[j][i] + R.m[i][j]) * t;
        c[k] = (R.m[k][i] + R.m[i][k]) * t;
        q.x = c[0]; q.y = c[1]; q.z = c[2];
    }
    return q;
}
// Euler ZYX update matrix of the GN step (src/ct_icp/ct_icp.cpp:916-932)
CT_HD M3 eulerZYX(double a, double b, double g) {
    M3 R;
    double ca = cos(a), sa = sin(a), cb = cos(b), sb = sin(b), cg = cos(g), sg = sin(g);
    R.m[0][0] = cg * cb; R.m[0][1] = -sg * ca + cg * sb * sa; R.m[0][2] = sg * sa + cg * sb * ca;
    R.m[1][0] = sg * cb; R.m[1][1] = cg * ca + sg * sb * sa;  R.m[1][2] = -cg * sa + sg * sb * ca;
    R.m[2][0] = -sb;     R.m[2][1] = cb * sa;                 R.m[2][2] = cb * ca;
    return R;
}

struct Se3 {   // slam::TSE3<double>
    Q4 q;
    V3 t;
};
CT_HD Se3 se3_identity() { return Se3{{0, 0, 0, 1}, {0, 0, 0}}; }
CT_HD Se3 se3_inverse(Se3 a) {   // types.h:327-332
    Se3 r;
    r.q = qinverse(a.q);
    V3 v = qrot(r.q, a.t);
    r.t = {-v.x, -v.y, -v.z};
    return r;
}
CT_HD Se3 se3_mul(Se3 a, Se3 b) {   // types.h:344-351
    Se3 r;
    r.q = qnormalized(qmul(a.q, b.q));
    r.t = qrot(qnormalized(a.q), b.t) + a.t;
    return r;
}
// world = Interpolate(begin, end, alpha) * raw  (types.h:361-366 then :354-357: slerp, lerp, quat.normalized()*p + tr)
CT_HD V3 ct_transform(Q4 qb, V3 tb, Q4 qe, V3 te, double alpha, V3 raw) {
    Q4 q = qnormalized(qslerp(qb, qe, alpha));
    V3 t = (1.0 - alpha) * tb + alpha * te;
    return qrot(q, raw) + t;
}
CT_HD V3 ct_transform_c(Q4 qb, V3 tb, Q4 qe, V3 te, double alpha, V3 raw, const SlerpConsts &c) {
    Q4 q = qslerp_c(qb, qe, alpha, c);
#ifdef __CUDA_ARCH__
    const double inv = rsqrt(qdot(q, q));   // one MUFU seed instead of sqrt + reciprocal (<= 1 ulp apart)
#else
    const double inv = 1.0 / sqrt(qdot(q, q));
#endif
    q = Q4{q.x * inv, q.y * inv, q.z * inv, q.w * inv};
    V3 t = (1.0 - alpha) * tb + alpha * te;
    return qrot(q, raw) + t;
}
#ifdef __CUDACC__
// ---- conversions without the XU pipe ---------------------------------------------------------------------------------
// F2F.F64.F32 / I2F.F64 / F2I.F64 and the 64-bit MUFU seeds of divisions and square roots execute on the XU pipe: few lanes
// per clock and a long latency, and every one of them sits ON the dependent chain of a keypoint (the gather kernels are
// bound by that chain, not by any pipe's throughput). The first round-2 build executed ~100 of them per
// keypoint-iteration; these helpers do the same conversions with integer / fp64-add instructions (exact, all values),
// which shortened the GN loop together with the polynomial sin / cos and the 1/n table:
// float → double: re-bias the exponent, shift the mantissa. Branch-free: fp32 denormals (|x| < 1.2e-38 — no coordinate or
// offset in metres is one) become zero, inf / nan become huge finite values (never inside a search radius).
__device__ __forceinline__ double f32_to_f64(float f) {
    const unsigned u = __float_as_uint(f);
    const unsigned mag = u & 0x7fffffffu;
    const bool tiny = mag < 0x00800000u;
    const unsigned hi = (u & 0x80000000u) | (tiny ? 0u : (mag >> 3) + 0x38000000u);
    return __hiloint2double((int) hi, tiny ? 0 : (int) (u << 29));
}
// int32 → double: 2^52 + 2^31 + i is exact, its low word is i ^ 0x80000000
__device__ __forceinline__ double i32_to_f64(int i) {
    return __hiloint2double(0x43300000, i ^ (int) 0x80000000) - 4503601774854144.0;
}
// floor of a double in [0, 2^31): rounding-down add of 2^52 leaves floor(x) in the low word
__device__ __forceinline__ int f64_floor_nonneg(double x) { return __double2loint(__dadd_rd(x, 4503599627370496.0)); }
// C truncation int(x) for |x| < 2^31
__device__ __forceinline__ int f64_trunc(double x) {
    const int k = f64_floor_nonneg(fabs(x));
    return x < 0.0 ? -k : k;
}

// A scan point lives on the device as fp32 (x, y, z, alpha) — what LiDAR drivers emit — plus an OPTIONAL residual plane
// `lo` = value - (double)(float)value (also fp32): hi + lo reproduces an fp64 input to ~2^-48 relative, i.e. exactly as far
// as voxel assignment and the 1e-4 m tolerance are concerned. lo == nullptr: the scan is float32-representable.
struct RawPoint {
    double x, y, z, alpha;
};
__device__ __forceinline__ RawPoint load_raw(const float4 *hi, const float4 *lo, size_t i) {
    const float4 h = hi[i];
    RawPoint r{f32_to_f64(h.x), f32_to_f64(h.y), f32_to_f64(h.z), f32_to_f64(h.w)};
    if (lo) {
        const float4 l = lo[i];
        r.x += (double) l.x; r.y += (double) l.y; r.z += (double) l.z; r.alpha += (double) l.w;
    }
    return r;
}
__device__ __forceinline__ void store_raw(float4 *hi, float4 *lo, size_t i, double x, double y, double z, double alpha) {
    const float4 h = make_float4((float) x, (float) y, (float) z, (float) alpha);
    hi[i] = h;
    if (lo) lo[i] = make_float4((float) (x - (double) h.x), (float) (y - (double) h.y), (float) (z - (double) h.z),
                                (float) (alpha - (double) h.w));
}
#endif

// slam::AngularDistance (types.h:141-156), degrees; returns NaN when the CHECK would fire
CT_HD double angular_distance_deg(Q4 a, Q4 b) {
    M3 Ra = qtoR(a), Rb = qtoR(b);
    double tr = 0;
    for (int i = 0; i < 3; ++i)
        for (int k = 0; k < 3; ++k) tr += Ra.m[i][k] * Rb.m[i][k];
    double n = (tr - 1.0) / 2.0;
    if (!(n < 1.0 + 1e-8 && n >= -1.0 - 1e-8)) return NAN;
    n = fmax(fmin(n, 1.0), -1.0);
    return acos(n) * (180.0 / M_PI);
}

// ---- order contract: counter-based permutation standing in for std::shuffle (DESIGN.md "Order contract") ----
CT_HD uint32_t mix32(uint32_t h) {
    h ^= h >> 16; h *= 0x85ebca6bu; h ^= h >> 13; h *= 0xc2b2ae35u; h ^= h >> 16;
    return h;
}
CT_HD uint64_t splitmix64(uint64_t x) {
    x += 0x9E3779B97F4A7C15ull;
    x = (x ^ (x >> 30)) * 0xBF58476D1CE4E5B9ull;
    x = (x ^ (x >> 27)) * 0x94D049BB133111EBull;
    return x ^ (x >> 31);
}
struct Perm {
    uint32_t n, half_bits, half_mask;
    uint32_t keys[4];
};
CT_HD Perm perm_make(uint64_t seed, uint64_t counter, uint32_t n) {
    Perm p;
    p.n = n;
    uint32_t bits = 2;
    while (bits < 32 && (uint64_t(1) << bits) < uint64_t(n)) bits += 2;
    p.half_bits = bits / 2;
    p.half_mask = (1u << p.half_bits) - 1u;
    uint64_t s = splitmix64(seed ^ splitmix64(counter));
    uint64_t s2 = splitmix64(s);
    p.keys[0] = uint32_t(s); p.keys[1] = uint32_t(s >> 32); p.keys[2] = uint32_t(s2); p.keys[3] = uint32_t(s2 >> 32);
    return p;
}
CT_HD uint32_t perm_apply(const Perm &p, uint32_t i) {
    uint32_t v = i;
    do {
        uint32_t l = v >> p.half_bits, r = v & p.half_mask;
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            uint32_t f = mix32(r ^ p.keys[k]) & p.half_mask;
            uint32_t nl = r;
            r = l ^ f;
            l = nl;
        }
        v = (l << p.half_bits) | r;
    } while (v >= p.n);
    return v;
}

}  // namespace cticp
