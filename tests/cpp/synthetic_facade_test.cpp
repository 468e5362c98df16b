// slam::Scene / SyntheticSensorAcquisition / ApplyUniformNoise of the C++ facade (ct_icp_b200/odometry.hpp) against the
// CPU restatement of the reference (tests/oracle_synthetic/orc_synthetic.cpp, linked in): Distance of every primitive,
// GeneratePoints(CloseToLocation), GeneratePoses, GenerateFrame(s), GenerateSensorPoints and ApplyUniformNoise on a
// seeded scene of every primitive kind along a turning trajectory.
// Exit 0 and "SYNTHETIC FACADE OK" on success; exit 42 when no device is usable (CTICP_ERR_NO_DEVICE); 1 on a mismatch.
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <random>
#include <vector>

#include "ct_icp_b200/odometry.hpp"

struct orc_synthetic_scene;
struct orc_trajectory;
extern "C" {
int orc_synthetic_scene_create(const double *, size_t, const double *, size_t, const double *, size_t, const double *,
                               size_t, int, orc_synthetic_scene **);
int orc_synthetic_scene_distance(orc_synthetic_scene *, const double *, size_t, double *);
int64_t orc_synthetic_generate_points(orc_synthetic_scene *, size_t, const double *, double, uint64_t, double *, size_t,
                                      uint32_t *);
int64_t orc_synthetic_generate_frames(orc_synthetic_scene *, orc_trajectory *, const cticp_synthetic_frame *, size_t,
                                      size_t, double, uint64_t, const cticp_cloud_sink *, uint32_t *, uint64_t *);
int64_t orc_synthetic_generate_poses(orc_trajectory *, double, cticp_pose *, size_t);
int orc_apply_uniform_noise(cticp_pose *, size_t, double, double, uint64_t);
int orc_trajectory_create(const cticp_pose *, size_t, int, orc_trajectory **);
}

namespace {
int failures = 0;
void expect(bool ok, const char *what, double a = 0, double b = 0) {
    if (!ok && failures++ < 20) std::printf("MISMATCH %s: %.17g vs %.17g\n", what, a, b);
}
bool close(double a, double b, double tol) { return std::fabs(a - b) <= tol; }
}  // namespace

int main() {
    std::mt19937_64 rng(20261018);
    std::uniform_real_distribution<double> u(-15.0, 15.0), r(0.1, 2.0);
    std::normal_distribution<double> nd(0.0, 1.0);
    slam::Scene scene;
    scene.seed = 77;
    std::vector<double> tri, lin, sph, bal;
    for (int i = 0; i < 30; ++i) {
        slam::Triangle::PointsArray a;
        for (auto &p : a)
            for (int k = 0; k < 3; ++k) p[k] = (i < 10 && k == 2) ? 0.0 : u(rng);   // the first ten: rank-2 floors
        scene.Triangles().emplace_back(a);
        for (auto &p : a) tri.insert(tri.end(), p.v, p.v + 3);
    }
    for (int i = 0; i < 10; ++i) {
        slam::Line::PointsArray a;
        for (auto &p : a)
            for (int k = 0; k < 3; ++k) p[k] = u(rng);
        scene.Lines().emplace_back(a);
        for (auto &p : a) lin.insert(lin.end(), p.v, p.v + 3);
    }
    for (int i = 0; i < 8; ++i) {
        const slam::Vec3d c{{u(rng), u(rng), u(rng)}};
        const double rs = r(rng), rb = r(rng);
        scene.Spheres().emplace_back(c, rs);
        scene.Balls().emplace_back(c, rb);
        sph.insert(sph.end(), {c[0], c[1], c[2], rs});
        bal.insert(bal.end(), {c[0], c[1], c[2], rb});
    }
    std::vector<slam::Pose> poses;
    std::vector<cticp_pose> cposes;
    for (int k = 0; k < 6; ++k) {
        slam::Pose p;
        double n = 0;
        for (int c = 0; c < 4; ++c) { p.pose.quat.c[c] = nd(rng); n += p.pose.quat.c[c] * p.pose.quat.c[c]; }
        for (int c = 0; c < 4; ++c) p.pose.quat.c[c] /= std::sqrt(n);
        for (int c = 0; c < 3; ++c) p.pose.tr[c] = 4.0 * nd(rng);
        p.dest_timestamp = k;
        p.dest_frame_id = (slam::frame_id_t) k;
        poses.push_back(p);
        cposes.push_back(ct_icp::detail::pose_to_c(p));
    }
    orc_synthetic_scene *os = nullptr;
    orc_trajectory *ot = nullptr;
    orc_synthetic_scene_create(tri.data(), 30, lin.data(), 10, sph.data(), 8, bal.data(), 8, 0, &os);
    orc_trajectory_create(cposes.data(), cposes.size(), 0, &ot);
    try {
        // Distance: the scene's batch and each primitive on its own, bit for bit
        std::vector<slam::Vec3d> q;
        for (int i = 0; i < 200; ++i) q.push_back(slam::Vec3d{{u(rng), u(rng), u(rng)}});
        q.push_back(scene.Triangles()[0].Points()[1]);
        const std::vector<double> d = scene.Distances(q);
        std::vector<double> od(d.size());
        orc_synthetic_scene_distance(os, q[0].v, q.size(), od.data());
        for (size_t i = 0; i < d.size(); ++i) expect(d[i] == od[i], "Scene distance", d[i], od[i]);
        const size_t np = scene.NumPrimitives();
        expect(scene.Triangles()[3].Distance(q[5]) == od[5 * np + 3], "Triangle::Distance");
        expect(scene.Lines()[2].Distance(q[6]) == od[6 * np + 32], "Line::Distance");
        expect(scene.Spheres()[1].Distance(q[7]) == od[7 * np + 41], "Sphere::Distance");
        expect(scene.Balls()[4].ComputeDistance(q[8]) == od[8 * np + 52], "Ball::ComputeDistance");
        expect(scene.Triangles()[0].Distance(q.back()) == 0.0, "Distance on a vertex");

        // GeneratePoints / GeneratePointsCloseToLocation
        for (int pass = 0; pass < 2; ++pass) {
            const slam::Vec3d loc{{1.0, -2.0, 0.5}};
            const auto pts = pass ? scene.GeneratePointsCloseToLocation(40, loc, 8.0) : scene.GeneratePoints(40);
            const int64_t n = orc_synthetic_generate_points(os, 40, pass ? loc.v : nullptr, 8.0, 77, nullptr, 0, nullptr);
            std::vector<double> o(3 * (size_t) n);
            orc_synthetic_generate_points(os, 40, pass ? loc.v : nullptr, 8.0, 77, o.data(), (size_t) n, nullptr);
            expect((int64_t) pts.size() == n && n > 0, "GeneratePoints count", (double) pts.size(), (double) n);
            for (size_t i = 0; i < pts.size() && (int64_t) i < n; ++i)
                for (int k = 0; k < 3; ++k) expect(close(pts[i][k], o[3 * i + k], 1e-12 * 16), "GeneratePoints");
        }

        // GeneratePoses and GenerateFrame(s) of a SyntheticSensorAcquisition
        auto shared = std::make_shared<slam::Scene>(scene);
        slam::SyntheticSensorAcquisition acq(shared, slam::LinearContinuousTrajectory::Create(std::vector<slam::Pose>(poses)));
        const std::vector<slam::Pose> sampled = acq.GeneratePoses(8.0);
        std::vector<cticp_pose> osampled(sampled.size() + 1);
        const int64_t ns = orc_synthetic_generate_poses(ot, 8.0, osampled.data(), osampled.size());
        expect(ns == (int64_t) sampled.size(), "GeneratePoses count", (double) sampled.size(), (double) ns);
        for (size_t i = 0; i < sampled.size() && (int64_t) i < ns; ++i) {
            expect(sampled[i].dest_timestamp == osampled[i].dest_timestamp, "GeneratePoses t");
            for (int k = 0; k < 3; ++k) expect(close(sampled[i].pose.tr[k], osampled[i].tr[k], 1e-12), "GeneratePoses tr");
        }
        std::vector<cticp_synthetic_frame> frames;
        for (size_t k = 0; k + 1 < sampled.size(); ++k)
            frames.push_back({sampled[k].dest_timestamp, sampled[k + 1].dest_timestamp, (uint32_t) k, 0});
        const std::vector<slam::WPoint3D> pts = acq.GenerateFrames(60, frames, 12.0);
        std::vector<double> raw, world;
        std::vector<uint64_t> ends(frames.size());
        for (int w = 0; w < 2; ++w) {
            std::vector<double> &buf = w ? world : raw;
            buf.resize(4 * pts.size() + 4);
            const cticp_cloud_sink sink{buf.data(), pts.size(), 32, 0, CTICP_DTYPE_FLOAT64, 24, CTICP_DTYPE_FLOAT64, w};
            const int64_t n = orc_synthetic_generate_frames(os, ot, frames.data(), frames.size(), 60, 12.0, 77, &sink,
                                                            nullptr, ends.data());
            expect(n == (int64_t) pts.size() && n > 1000, "GenerateFrames count", (double) pts.size(), (double) n);
        }
        size_t k = 0;
        for (size_t i = 0; i < pts.size(); ++i) {
            while (k < frames.size() && ends[k] <= i) ++k;
            expect(pts[i].index_frame == frames[k].frame_id, "index_frame", pts[i].index_frame, frames[k].frame_id);
            expect(pts[i].Timestamp() == raw[4 * i + 3], "timestamp", pts[i].Timestamp(), raw[4 * i + 3]);
            for (int c = 0; c < 3; ++c) {
                expect(close(pts[i].RawPoint()[c], raw[4 * i + c], 1e-12 * 32), "raw", pts[i].RawPoint()[c], raw[4 * i + c]);
                expect(close(pts[i].WorldPoint()[c], world[4 * i + c], 1e-12 * 32), "world");
            }
        }
        // GenerateFrame of one frame is that frame's slice; GenerateSensorPoints between the same two poses is the same
        const size_t f = frames.size() / 2;
        const auto one = acq.GenerateFrame(60, frames[f].begin_ts, frames[f].end_ts, frames[f].frame_id, 12.0);
        expect(one.size() == ends[f] - ends[f - 1], "GenerateFrame size");
        slam::Pose b = sampled[f], e = sampled[f + 1];
        b.dest_frame_id = (slam::frame_id_t) f;
        const auto sensor = shared->GenerateSensorPoints(60, b, e, 12.0);
        expect(sensor.size() == one.size(), "GenerateSensorPoints size", (double) sensor.size(), (double) one.size());
        for (size_t i = 0; i < one.size() && i < sensor.size(); ++i) {
            expect(std::memcmp(&one[i], &pts[ends[f - 1] + i], sizeof(slam::WPoint3D)) == 0, "GenerateFrame bytes");
            expect(std::memcmp(&one[i], &sensor[i], sizeof(slam::WPoint3D)) == 0, "GenerateSensorPoints bytes");
        }
    } catch (const ct_icp::CticpFailure &e) {
        std::printf("%s\n", e.what());
        return e.code == CTICP_ERR_NO_DEVICE ? 42 : 1;
    }

    // ApplyUniformNoise
    std::vector<slam::Pose> noisy = poses;
    slam::ApplyUniformNoise(noisy, 2.0, 0.1, 5);
    orc_apply_uniform_noise(cposes.data(), cposes.size(), 2.0, 0.1, 5);
    for (size_t i = 0; i < noisy.size(); ++i)
        for (int c = 0; c < 3; ++c) expect(close(noisy[i].pose.tr[c], cposes[i].tr[c], 1e-14), "ApplyUniformNoise");
    const slam::SE3 single = slam::ApplyUniformNoise(poses[0].pose, 2.0, 0.1, 5);
    for (int c = 0; c < 4; ++c) expect(single.quat.c[c] == noisy[0].pose.quat.c[c], "ApplyUniformNoise(SE3)");

    if (failures) {
        std::printf("%d mismatches\n", failures);
        return 1;
    }
    std::printf("SYNTHETIC FACADE OK\n");
    return 0;
}
