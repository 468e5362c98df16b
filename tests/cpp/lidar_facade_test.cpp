// slam::LidarScene of the C++ facade (ct_icp_b200/odometry.hpp) against the host caster tools/raycast.c (linked in):
// Raycast of random rays on a seeded scene of solid boxes and cylinders bit for bit, and GenerateSweeps of a 16-ring
// sensor along a two-pose trajectory: counts, keep bounds, frame ids, raw = world seen from the column's pose, and a
// frame alone equal to the same frame in a batch.
// Exit 0 and "LIDAR FACADE OK" on success; exit 42 when no device is usable (CTICP_ERR_NO_DEVICE); 1 on a mismatch.
#include <cmath>
#include <cstdio>
#include <cstring>
#include <random>
#include <vector>

#include "ct_icp_b200/odometry.hpp"

extern "C" void raycast_scene(const double *o, const double *d, size_t n, const double *boxes, size_t nb,
                              const double *cyl, size_t nc, double max_range, uint64_t seed, double *out);

namespace {
int failures = 0;
void expect(bool ok, const char *what, double a = 0, double b = 0) {
    if (!ok && failures++ < 20) std::printf("MISMATCH %s: %.17g vs %.17g\n", what, a, b);
}
}  // namespace

int main() {
    std::mt19937_64 rng(20261018);
    std::uniform_real_distribution<double> u(-40.0, 40.0), s(0.3, 8.0), z(0.0, 2.0);
    std::vector<std::array<double, 7>> boxes;
    std::vector<std::array<double, 4>> cyl;
    for (int i = 0; i < 120; ++i) {
        const double x = u(rng), y = u(rng), z0 = z(rng);
        boxes.push_back({x, y, z0, x + s(rng), y + s(rng), z0 + s(rng), 0.0});
    }
    for (int i = 0; i < 30; ++i) cyl.push_back({u(rng), u(rng), 0.1 * s(rng), s(rng)});
    try {
        const slam::LidarScene scene(boxes, cyl);
        std::vector<slam::Vec3d> o(20000), d(20000);
        std::normal_distribution<double> nd(0.0, 1.0);
        for (size_t i = 0; i < o.size(); ++i) {
            o[i] = slam::Vec3d{{u(rng), u(rng), 0.5 + z(rng)}};
            double v[3] = {nd(rng), nd(rng), 0.2 * nd(rng)}, n = std::sqrt(v[0] * v[0] + v[1] * v[1] + v[2] * v[2]);
            d[i] = slam::Vec3d{{v[0] / n, v[1] / n, v[2] / n}};
        }
        const std::vector<double> got = scene.Raycast(o, d, 50.0, 99);
        std::vector<double> want(o.size());
        raycast_scene(o[0].v, d[0].v, o.size(), boxes[0].data(), boxes.size(), cyl[0].data(), cyl.size(), 50.0, 99,
                      want.data());
        for (size_t i = 0; i < got.size(); ++i)
            expect(std::memcmp(&got[i], &want[i], sizeof(double)) == 0, "Raycast", got[i], want[i]);

        std::vector<slam::Pose> poses(2);
        for (int k = 0; k < 2; ++k) {
            poses[k].pose.tr[0] = -5.0 + 10.0 * k;
            poses[k].pose.tr[2] = 1.7;
            poses[k].dest_timestamp = k;
            poses[k].dest_frame_id = 0;
        }
        const slam::LinearContinuousTrajectory traj = slam::LinearContinuousTrajectory::Create(std::move(poses));
        slam::LidarSensor sensor;
        for (int r = 0; r < 16; ++r) sensor.elevations_deg.push_back(15.0 - 2.0 * r);
        sensor.n_azimuth = 900;
        sensor.min_range = 1.0;
        sensor.max_range = 60.0;
        const std::vector<cticp_lidar_frame> frames{{0.1, 1, 0}, {0.5, 5, 0}, {0.8, 8, 0}};
        std::vector<uint64_t> ends;
        const std::vector<slam::WPoint3D> pts = scene.GenerateSweeps(traj, sensor, frames, 3, &ends);
        expect(ends.size() == 3 && ends[2] == pts.size() && pts.size() > 5000, "GenerateSweeps count", pts.size());
        size_t k = 0;
        for (size_t i = 0; i < pts.size(); ++i) {
            while (i >= ends[k]) ++k;
            const slam::Vec3d &p = pts[i].RawPoint();
            const double r = std::sqrt(p[0] * p[0] + p[1] * p[1] + p[2] * p[2]);
            expect(r > sensor.min_range - 1e-9 && r < sensor.max_range + 1e-9, "keep bounds", r);
            expect(pts[i].index_frame == frames[k].frame_id, "index_frame", pts[i].index_frame, frames[k].frame_id);
            // the trajectory translates along x without turning: world = raw + the column's position
            const double t = pts[i].raw_point.timestamp, x = -5.0 + 10.0 * t;
            expect(std::fabs(pts[i].WorldPoint()[0] - (p[0] + x)) < 1e-9, "world x", pts[i].WorldPoint()[0], p[0] + x);
            expect(std::fabs(pts[i].WorldPoint()[2] - (p[2] + 1.7)) < 1e-9, "world z", pts[i].WorldPoint()[2], p[2] + 1.7);
        }
        const std::vector<slam::WPoint3D> one = scene.GenerateSweeps(traj, sensor, {frames[1]}, 3);
        expect(one.size() == ends[1] - ends[0], "GenerateSweeps alone", one.size(), ends[1] - ends[0]);
        for (size_t i = 0; i < one.size() && ends[0] + i < pts.size(); ++i)
            expect(std::memcmp(&one[i], &pts[ends[0] + i], sizeof(slam::WPoint3D)) == 0, "GenerateSweeps bytes");
    } catch (const ct_icp::CticpFailure &e) {
        std::printf("%s\n", e.what());
        return e.code == CTICP_ERR_NO_DEVICE ? 42 : 1;
    }
    if (failures) {
        std::printf("%d mismatches\n", failures);
        return 1;
    }
    std::printf("LIDAR FACADE OK\n");
    return 0;
}
