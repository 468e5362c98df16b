// orc_dataset.cpp — dependency-free CPU restatement of the reference's dataset readers (src/ct_icp/dataset.cpp,
// src/SlamCore/io.cxx), written the way the reference is, not the way the engine is: TEST INFRASTRUCTURE.
//   - NCLTIterator::NextBatch / DoNext read the bytes through a std::istream, field by field;
//   - kitti_frame_filter goes through small fixed-size matrix types whose operations follow Eigen 3's evaluators:
//     cross (cross_impl), squaredNorm (a redux in index order), normalize (divide by sqrt), AngleAxis::toRotationMatrix,
//     and a coefficient-based matrix-vector product (sum over k in order);
//   - LoadPosesKITTIFormat and the HILTI reader extract values with `std::istream >> double`, NCLT rows with std::stod;
//     the calibration is inverted with the general cofactor inverse of a 4x4 matrix, as Matrix4d::inverse() is.
// Built with -ffp-contract=off (tests/oracle_dataset_lib.py).
#include <algorithm>
#include <cmath>
#include <cstdint>
#include <cstring>
#include <sstream>
#include <string>
#include <vector>

namespace {

template <int R, int C>
struct Mat {
    double a[R][C] = {};
    double &operator()(int i, int j) { return a[i][j]; }
    double operator()(int i, int j) const { return a[i][j]; }
    static Mat Identity() {
        Mat m;
        for (int i = 0; i < R && i < C; ++i) m.a[i][i] = 1.0;
        return m;
    }
};
using V3 = Mat<3, 1>;
using M3 = Mat<3, 3>;
using M4 = Mat<4, 4>;

template <int R, int K, int C>
Mat<R, C> operator*(const Mat<R, K> &l, const Mat<K, C> &r) {   // coefficient-based: sum over k, in order
    Mat<R, C> o;
    for (int i = 0; i < R; ++i)
        for (int j = 0; j < C; ++j) {
            double s = l(i, 0) * r(0, j);
            for (int k = 1; k < K; ++k) s = s + l(i, k) * r(k, j);
            o(i, j) = s;
        }
    return o;
}
V3 vec(double x, double y, double z) {
    V3 v;
    v(0, 0) = x, v(1, 0) = y, v(2, 0) = z;
    return v;
}
V3 cross(const V3 &a, const V3 &b) {   // Eigen cross_impl
    return vec(a(1, 0) * b(2, 0) - a(2, 0) * b(1, 0), a(2, 0) * b(0, 0) - a(0, 0) * b(2, 0),
               a(0, 0) * b(1, 0) - a(1, 0) * b(0, 0));
}
double squaredNorm(const V3 &v) {   // redux of cwiseAbs2, index order
    double s = v(0, 0) * v(0, 0);
    for (int i = 1; i < 3; ++i) s = s + v(i, 0) * v(i, 0);
    return s;
}
void normalize(V3 &v) {   // MatrixBase::normalize: z = squaredNorm(); if (z > 0) *this /= sqrt(z)
    const double z = squaredNorm(v);
    if (z > 0.0) {
        const double s = std::sqrt(z);
        for (int i = 0; i < 3; ++i) v(i, 0) = v(i, 0) / s;
    }
}
M3 angle_axis_matrix(double angle, const V3 &axis) {   // AngleAxis::toRotationMatrix
    M3 res;
    V3 sin_axis, cos1_axis;
    const double s = std::sin(angle), c = std::cos(angle);
    for (int i = 0; i < 3; ++i) {
        sin_axis(i, 0) = s * axis(i, 0);
        cos1_axis(i, 0) = (1.0 - c) * axis(i, 0);
    }
    double tmp = cos1_axis(0, 0) * axis(1, 0);
    res(0, 1) = tmp - sin_axis(2, 0);
    res(1, 0) = tmp + sin_axis(2, 0);
    tmp = cos1_axis(0, 0) * axis(2, 0);
    res(0, 2) = tmp + sin_axis(1, 0);
    res(2, 0) = tmp - sin_axis(1, 0);
    tmp = cos1_axis(1, 0) * axis(2, 0);
    res(1, 2) = tmp - sin_axis(0, 0);
    res(2, 1) = tmp + sin_axis(0, 0);
    for (int i = 0; i < 3; ++i) res(i, i) = cos1_axis(i, 0) * axis(i, 0) + c;
    return res;
}

// ---- quaternions (x, y, z, w) ----
struct Q {
    double x = 0, y = 0, z = 0, w = 1;
};
Q qmul(const Q &a, const Q &b) {
    return {a.w * b.x + a.x * b.w + a.y * b.z - a.z * b.y, a.w * b.y + a.y * b.w + a.z * b.x - a.x * b.z,
            a.w * b.z + a.z * b.w + a.x * b.y - a.y * b.x, a.w * b.w - a.x * b.x - a.y * b.y - a.z * b.z};
}
double qnorm(const Q &q) { return std::sqrt(q.x * q.x + q.y * q.y + q.z * q.z + q.w * q.w); }
Q qnormalized(const Q &q) {
    const double n = qnorm(q);
    return {q.x / n, q.y / n, q.z / n, q.w / n};
}
Q qinverse(const Q &q) {
    const double n2 = q.x * q.x + q.y * q.y + q.z * q.z + q.w * q.w;
    return {-q.x / n2, -q.y / n2, -q.z / n2, q.w / n2};
}
M3 qmatrix(const Q &q) {   // Quaternion::toRotationMatrix
    M3 r;
    const double tx = 2 * q.x, ty = 2 * q.y, tz = 2 * q.z;
    const double twx = tx * q.w, twy = ty * q.w, twz = tz * q.w, txx = tx * q.x, txy = ty * q.x, txz = tz * q.x;
    const double tyy = ty * q.y, tyz = tz * q.y, tzz = tz * q.z;
    r(0, 0) = 1 - (tyy + tzz), r(0, 1) = txy - twz, r(0, 2) = txz + twy;
    r(1, 0) = txy + twz, r(1, 1) = 1 - (txx + tzz), r(1, 2) = tyz - twx;
    r(2, 0) = txz - twy, r(2, 1) = tyz + twx, r(2, 2) = 1 - (txx + tyy);
    return r;
}
Q qfrommatrix(const M3 &m) {   // Quaternion(Matrix3): quaternionbase_assign_impl
    Q q;
    double t = m(0, 0) + m(1, 1) + m(2, 2);
    if (t > 0) {
        t = std::sqrt(t + 1.0);
        q.w = 0.5 * t;
        t = 0.5 / t;
        q.x = (m(2, 1) - m(1, 2)) * t, q.y = (m(0, 2) - m(2, 0)) * t, q.z = (m(1, 0) - m(0, 1)) * t;
    } else {
        int i = 0;
        if (m(1, 1) > m(0, 0)) i = 1;
        if (m(2, 2) > m(i, i)) i = 2;
        const int j = (i + 1) % 3, k = (j + 1) % 3;
        t = std::sqrt(m(i, i) - m(j, j) - m(k, k) + 1.0);
        double c[3];
        c[i] = 0.5 * t;
        t = 0.5 / t;
        q.w = (m(k, j) - m(j, k)) * t;
        c[j] = (m(j, i) + m(i, j)) * t;
        c[k] = (m(k, i) + m(i, k)) * t;
        q.x = c[0], q.y = c[1], q.z = c[2];
    }
    return q;
}
V3 qrot(const Q &q, const V3 &v) {   // _transformVector
    const V3 qv = vec(q.x, q.y, q.z);
    V3 uv = cross(qv, v);
    for (int i = 0; i < 3; ++i) uv(i, 0) = uv(i, 0) + uv(i, 0);
    const V3 c = cross(qv, uv);
    return vec(v(0, 0) + q.w * uv(0, 0) + c(0, 0), v(1, 0) + q.w * uv(1, 0) + c(1, 0), v(2, 0) + q.w * uv(2, 0) + c(2, 0));
}
struct SE3 {   // slam::TSE3
    Q quat;
    V3 tr;
    SE3 Inverse() const {
        SE3 r;
        r.quat = qinverse(quat);
        const V3 v = qrot(r.quat, tr);
        r.tr = vec(-v(0, 0), -v(1, 0), -v(2, 0));
        return r;
    }
    SE3 operator*(const SE3 &b) const {
        SE3 r;
        r.quat = qnormalized(qmul(quat, b.quat));
        const V3 v = qrot(qnormalized(quat), b.tr);
        r.tr = vec(v(0, 0) + tr(0, 0), v(1, 0) + tr(1, 0), v(2, 0) + tr(2, 0));
        return r;
    }
    M4 Matrix() const {
        M4 m = M4::Identity();
        const M3 r = qmatrix(quat);
        for (int i = 0; i < 3; ++i) {
            for (int j = 0; j < 3; ++j) m(i, j) = r(i, j);
            m(i, 3) = tr(i, 0);
        }
        return m;
    }
};
SE3 se3(Q q, V3 t) { return SE3{qnormalized(q), t}; }   // TSE3(quat, tr) normalises
Q qaxis(double angle, int axis) {   // Quaternion(AngleAxis)
    Q q;
    q.w = std::cos(0.5 * angle);
    const double s = std::sin(0.5 * angle);
    (axis == 0 ? q.x : axis == 1 ? q.y : q.z) = s;
    return q;
}
M3 ypr(double yaw, double pitch, double roll) {
    return qmatrix(qmul(qmul(qaxis(yaw, 2), qaxis(pitch, 1)), qaxis(roll, 0)));
}
M4 inverse4(const M4 &m) {   // the general inverse: adjugate / determinant
    double a[16], inv[16];
    for (int i = 0; i < 16; ++i) a[i] = m(i / 4, i % 4);
    inv[0] = a[5] * a[10] * a[15] - a[5] * a[11] * a[14] - a[9] * a[6] * a[15] + a[9] * a[7] * a[14] + a[13] * a[6] * a[11] - a[13] * a[7] * a[10];
    inv[4] = -a[4] * a[10] * a[15] + a[4] * a[11] * a[14] + a[8] * a[6] * a[15] - a[8] * a[7] * a[14] - a[12] * a[6] * a[11] + a[12] * a[7] * a[10];
    inv[8] = a[4] * a[9] * a[15] - a[4] * a[11] * a[13] - a[8] * a[5] * a[15] + a[8] * a[7] * a[13] + a[12] * a[5] * a[11] - a[12] * a[7] * a[9];
    inv[12] = -a[4] * a[9] * a[14] + a[4] * a[10] * a[13] + a[8] * a[5] * a[14] - a[8] * a[6] * a[13] - a[12] * a[5] * a[10] + a[12] * a[6] * a[9];
    inv[1] = -a[1] * a[10] * a[15] + a[1] * a[11] * a[14] + a[9] * a[2] * a[15] - a[9] * a[3] * a[14] - a[13] * a[2] * a[11] + a[13] * a[3] * a[10];
    inv[5] = a[0] * a[10] * a[15] - a[0] * a[11] * a[14] - a[8] * a[2] * a[15] + a[8] * a[3] * a[14] + a[12] * a[2] * a[11] - a[12] * a[3] * a[10];
    inv[9] = -a[0] * a[9] * a[15] + a[0] * a[11] * a[13] + a[8] * a[1] * a[15] - a[8] * a[3] * a[13] - a[12] * a[1] * a[11] + a[12] * a[3] * a[9];
    inv[13] = a[0] * a[9] * a[14] - a[0] * a[10] * a[13] - a[8] * a[1] * a[14] + a[8] * a[2] * a[13] + a[12] * a[1] * a[10] - a[12] * a[2] * a[9];
    inv[2] = a[1] * a[6] * a[15] - a[1] * a[7] * a[14] - a[5] * a[2] * a[15] + a[5] * a[3] * a[14] + a[13] * a[2] * a[7] - a[13] * a[3] * a[6];
    inv[6] = -a[0] * a[6] * a[15] + a[0] * a[7] * a[14] + a[4] * a[2] * a[15] - a[4] * a[3] * a[14] - a[12] * a[2] * a[7] + a[12] * a[3] * a[6];
    inv[10] = a[0] * a[5] * a[15] - a[0] * a[7] * a[13] - a[4] * a[1] * a[15] + a[4] * a[3] * a[13] + a[12] * a[1] * a[7] - a[12] * a[3] * a[5];
    inv[14] = -a[0] * a[5] * a[14] + a[0] * a[6] * a[13] + a[4] * a[1] * a[14] - a[4] * a[2] * a[13] - a[12] * a[1] * a[6] + a[12] * a[2] * a[5];
    inv[3] = -a[1] * a[6] * a[11] + a[1] * a[7] * a[10] + a[5] * a[2] * a[11] - a[5] * a[3] * a[10] - a[9] * a[2] * a[7] + a[9] * a[3] * a[6];
    inv[7] = a[0] * a[6] * a[11] - a[0] * a[7] * a[10] - a[4] * a[2] * a[11] + a[4] * a[3] * a[10] + a[8] * a[2] * a[7] - a[8] * a[3] * a[6];
    inv[11] = -a[0] * a[5] * a[11] + a[0] * a[7] * a[9] + a[4] * a[1] * a[11] - a[4] * a[3] * a[9] - a[8] * a[1] * a[7] + a[8] * a[3] * a[5];
    inv[15] = a[0] * a[5] * a[10] - a[0] * a[6] * a[9] - a[4] * a[1] * a[10] + a[4] * a[2] * a[9] + a[8] * a[1] * a[6] - a[8] * a[2] * a[5];
    const double det = a[0] * inv[0] + a[1] * inv[4] + a[2] * inv[8] + a[3] * inv[12];
    M4 r;
    for (int i = 0; i < 16; ++i) r(i / 4, i % 4) = inv[i] / det;
    return r;
}
M3 rows(const double *v) {
    M3 m;
    for (int i = 0; i < 9; ++i) m(i / 3, i % 3) = v[i];
    return m;
}

struct Pose {
    SE3 pose;
    double dest_timestamp = -1;
    uint32_t dest_frame_id = 0xFFFFFFFFu;
};

}  // namespace

extern "C" {

// DoNext over every frame: xyz[3 count] and t[count] (when cap allows), frame_ends[frames]; returns the point count,
// *frames the frame count; -1 for a bad magic or (final) a truncated packet
int64_t orc_nclt_decode(const unsigned char *bytes, size_t n, uint32_t A, int final, double *xyz, double *t, size_t cap,
                        uint64_t *frame_ends, size_t fcap, int64_t *frames) {
    std::istringstream file(std::string(reinterpret_cast<const char *>(bytes), n));
    std::vector<std::vector<double>> pkt_xyz;
    std::vector<double> pkt_t;
    std::vector<uint32_t> pkt_n;
    while ((size_t) file.tellg() < n) {   // NextBatch, ending after the last complete packet
        const size_t off = (size_t) file.tellg();
        unsigned short magic[4];
        if (n - off < 8) {   // a partial header: the end of a chunk, or a truncated stream
            if (final) return -1;
            break;
        }
        file.read(reinterpret_cast<char *>(magic), 8);
        for (unsigned short m : magic)
            if (m != 44444) return -1;
        if (n - off < 24) {
            if (final) return -1;
            break;
        }
        unsigned int num_hits, padding;
        unsigned long long utime;
        file.read(reinterpret_cast<char *>(&num_hits), 4);
        file.read(reinterpret_cast<char *>(&utime), 8);
        file.read(reinterpret_cast<char *>(&padding), 4);
        if (off + 24 + 8ull * num_hits > n) {
            if (final) return -1;
            break;
        }
        std::vector<double> pts(3 * (size_t) num_hits);
        unsigned short xyz_u[3];
        unsigned char il[2];
        for (unsigned pid = 0; pid < num_hits; ++pid) {
            file.read(reinterpret_cast<char *>(xyz_u), sizeof(xyz_u));
            file.read(reinterpret_cast<char *>(il), sizeof(il));
            pts[3 * pid] = ((double) xyz_u[0]) * 0.005 - 100.0;
            pts[3 * pid + 1] = ((double) xyz_u[1]) * 0.005 - 100.0;
            pts[3 * pid + 2] = ((double) xyz_u[2]) * 0.005 - 100.0;
        }
        pkt_xyz.push_back(std::move(pts));
        pkt_t.push_back((double) utime);
        pkt_n.push_back(num_hits);
    }
    const size_t P = pkt_n.size(), F = final ? (P + A - 1) / A : P / A;
    int64_t count = 0;
    for (size_t f = 0; f < F; ++f) {
        for (size_t p = f * A; p < std::min(P, (f + 1) * A); ++p)
            for (uint32_t h = 0; h < pkt_n[p]; ++h, ++count)
                if ((size_t) count < cap) {
                    for (int k = 0; k < 3; ++k) xyz[3 * count + k] = pkt_xyz[p][3 * h + k];
                    t[count] = pkt_t[p];
                }
        if (f < fcap) frame_ends[f] = (uint64_t) count;
    }
    *frames = (int64_t) F;
    return count;
}

// kitti_frame_filter, dataset.cpp:85-110, in place on n fp64 points
void orc_kitti_frame_filter(double *xyz, size_t n) {
    const double KITTI_MIN_Z = -5.0, KITTI_GLOBAL_VERTICAL_ANGLE_OFFSET = 0.205;
    const V3 uz = vec(0., 0., 1.);
    for (size_t i = 0; i < n; ++i) {
        V3 old_pt = vec(xyz[3 * i], xyz[3 * i + 1], xyz[3 * i + 2]);
        if (old_pt(2, 0) > KITTI_MIN_Z) {
            V3 rotationVector = cross(old_pt, uz);
            normalize(rotationVector);
            const M3 rotationScan = angle_axis_matrix(KITTI_GLOBAL_VERTICAL_ANGLE_OFFSET * M_PI / 180.0, rotationVector);
            old_pt = rotationScan * old_pt;
        } else {
            old_pt = vec(0, 0, 0);
        }
        for (int k = 0; k < 3; ++k) xyz[3 * i + k] = old_pt(k, 0);
    }
}

// LoadPoses (dataset.cpp:998-1098) into out[cap][9]: qx qy qz qw tx ty tz dest_timestamp dest_frame_id; the count,
// -1 for a malformed NCLT row or an unknown dataset
int64_t orc_ground_truth(int dataset, int sequence_id, const char *text, size_t n, double *out, size_t cap) {
    std::istringstream file(std::string(text, n));
    std::vector<Pose> poses;
    std::string line;
    M4 Calib = M4::Identity();
    static const double KITTI_R[3][9] = {
        {4.276802385584e-04, -9.999672484946e-01, -8.084491683471e-03, -7.210626507497e-03, 8.081198471645e-03,
         -9.999413164504e-01, 9.999738645903e-01, 4.859485810390e-04, -7.206933692422e-03},
        {2.347736981471e-04, -9.999441545438e-01, -1.056347781105e-02, 1.044940741659e-02, 1.056535364138e-02,
         -9.998895741176e-01, 9.999453885620e-01, 1.243653783865e-04, 1.045130299567e-02},
        {-1.857739385241e-03, -9.999659513510e-01, -8.039975204516e-03, -6.481465826011e-03, 8.051860151134e-03,
         -9.999466081774e-01, 9.999773098287e-01, -1.805528627661e-03, -6.496203536139e-03}};
    static const double KITTI_T[3][3] = {{-1.198459927713e-02, -5.403984729748e-02, -2.921968648686e-01},
                                         {-2.796816941295e-03, -7.510879138296e-02, -2.721327964059e-01},
                                         {-4.784029760483e-03, -7.337429464231e-02, -3.339968064433e-01}};
    if (dataset == 5 || dataset == 6) {   // ReadHILTIPosesInLidarFrame
        const SE3 l2i = dataset == 5 ? se3(qnormalized(Q{0.999993918507834, 0.0012283821413574625,
                                                         -0.0032596475280467258, -0.00016947759535612024}),
                                           vec(0.01001966915517371, -0.006645473484212856, 0.09473042428051345))
                                     : se3(qnormalized(Q{0.7071068, -0.7071068, 0, 0}), vec(-0.001, -0.00855, 0.055));
        const SE3 i2l = l2i.Inverse();
        while (std::getline(file, line)) {
            std::stringstream ls(line);
            Pose p;
            ls >> p.dest_timestamp >> p.pose.tr(0, 0) >> p.pose.tr(1, 0) >> p.pose.tr(2, 0) >> p.pose.quat.x >>
                p.pose.quat.y >> p.pose.quat.z >> p.pose.quat.w;
            p.pose = i2l * p.pose * l2i;
            poses.push_back(p);
        }
    } else if (dataset == 4) {   // ReadNCLTPoses
        bool have_init = false;
        SE3 init;
        while (std::getline(file, line)) {
            std::vector<std::string> tokens;
            while (!line.empty()) {
                auto it = line.find_first_of(',');
                if (it == std::string::npos) {
                    tokens.push_back(line);
                    line.clear();
                    break;
                }
                tokens.push_back(line.substr(0, it));
                line = line.substr(it + 1);
            }
            if (tokens.size() != 7) return -1;
            double v[7];
            try {
                for (int k = 0; k < 7; ++k) v[k] = std::stod(tokens[k]);
            } catch (...) {
                return -1;
            }
            Pose p;
            p.dest_timestamp = v[0];
            p.pose.tr = vec(v[1], v[2], v[3]);
            p.pose.quat = qfrommatrix(ypr(v[6], v[5], v[4]));
            const double nq = qnorm(p.pose.quat), nt = std::sqrt(squaredNorm(p.pose.tr));
            if (nq != nq || nt != nt) continue;
            if (!have_init) init = p.pose, have_init = true;
            p.pose = init.Inverse() * p.pose;
            poses.push_back(p);
        }
        M4 D = M4::Identity();
        const M3 r = ypr((-90.703 / 180.) * M_PI, (0.166 / 180.) * M_PI, (0.807 / 180.) * M_PI);
        for (int i = 0; i < 3; ++i)
            for (int j = 0; j < 3; ++j) D(i, j) = r(i, j);
        D(0, 3) = 0.002, D(1, 3) = -0.004, D(2, 3) = -0.957;
        Calib = D;
    } else if (dataset >= 0 && dataset <= 3) {   // LoadPosesKITTIFormat
        while (std::getline(file, line)) {
            if (line.empty()) continue;
            std::stringstream ss(line);
            M4 P = M4::Identity();
            ss >> P(0, 0) >> P(0, 1) >> P(0, 2) >> P(0, 3) >> P(1, 0) >> P(1, 1) >> P(1, 2) >> P(1, 3) >> P(2, 0) >>
                P(2, 1) >> P(2, 2) >> P(2, 3);
            Pose p;
            M3 R;
            for (int i = 0; i < 3; ++i)
                for (int j = 0; j < 3; ++j) R(i, j) = P(i, j);
            p.pose.quat = qfrommatrix(R);
            p.pose.tr = vec(P(0, 3), P(1, 3), P(2, 3));
            poses.push_back(p);
        }
        if (dataset == 0 || dataset == 2) {
            if (sequence_id < 0 || sequence_id > 21) return -1;
            const int c = sequence_id <= 2 ? 0 : sequence_id == 3 ? 1 : 2;
            Calib = se3(qfrommatrix(rows(KITTI_R[c])), vec(KITTI_T[c][0], KITTI_T[c][1], KITTI_T[c][2])).Matrix();
        } else if (dataset == 3) {
            const double R360[9] = {9.999290633685804508e-01,  5.805355888196038310e-03,  1.040029024212630118e-02,
                                    5.774300279226996999e-03,  -9.999787876452227442e-01, 3.013573682642321436e-03,
                                    1.041756443854582707e-02, -2.953305511449066945e-03, -9.999413744330052367e-01};
            Calib = se3(qfrommatrix(rows(R360)),
                        vec(-7.640302229235816922e-01, 2.966030253893782165e-01, -8.433819635885287935e-01)).Matrix();
        }
    } else {
        return -1;
    }
    if (dataset <= 4) {   // transform_poses
        const M4 CalibI = inverse4(Calib);
        int i = 0;
        for (Pose &p : poses) {
            const M4 mat = CalibI * p.pose.Matrix() * Calib;
            M3 R;
            for (int a = 0; a < 3; ++a)
                for (int b = 0; b < 3; ++b) R(a, b) = mat(a, b);
            p.pose.quat = qnormalized(qfrommatrix(R));
            p.pose.tr = vec(mat(0, 3), mat(1, 3), mat(2, 3));
            if (dataset == 0 || dataset == 2 || dataset == 3) {
                p.dest_timestamp = (static_cast<double>(i) + 0.5) * 0.1;
                p.dest_frame_id = i++;
            } else if (dataset == 1) {
                p.dest_timestamp = (static_cast<double>(i)) * 0.1;
                p.dest_frame_id = i++;
            }
        }
    }
    for (size_t k = 0; k < poses.size() && k < cap; ++k) {
        const Pose &p = poses[k];
        const double v[9] = {p.pose.quat.x, p.pose.quat.y, p.pose.quat.z, p.pose.quat.w, p.pose.tr(0, 0),
                             p.pose.tr(1, 0), p.pose.tr(2, 0), p.dest_timestamp, (double) p.dest_frame_id};
        std::memcpy(out + 9 * k, v, sizeof(v));
    }
    return (int64_t) poses.size();
}

}  // extern "C"
