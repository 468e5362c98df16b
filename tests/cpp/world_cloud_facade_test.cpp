// slam::SamplePointsInGrid and slam::WorldCloud of the C++ facade (ct_icp_b200/odometry.hpp) against the CPU
// restatement of the reference (tests/oracle_grid): the one-shot function, and a cloud grown in three adds.
// Exit 0 and "WORLD CLOUD FACADE OK" on success; exit 42 when no device is usable (CTICP_ERR_NO_DEVICE); 1 on a mismatch.
#include <cstdio>
#include <cstdlib>
#include <random>
#include <vector>

#include "ct_icp_b200/odometry.hpp"

extern "C" int64_t orc_sample_points_in_grid(int, const cticp_grid_sampling_options *, const double *, size_t, size_t,
                                             uint64_t *, size_t);

namespace {
std::vector<uint64_t> Oracle(const std::vector<slam::Vec3d> &pts, const slam::GridSamplingOptions &o) {
    cticp_grid_sampling_options c{};
    c.grid_size = o.grid_size;
    c.num_points_per_voxel = o.num_points_per_voxel;
    c.max_num_points = o.max_num_points;
    std::vector<uint64_t> out(pts.size() + 1);
    const int64_t n = orc_sample_points_in_grid(0, &c, pts[0].v, sizeof(slam::Vec3d), pts.size(), out.data(), out.size());
    out.resize((size_t) n);
    return out;
}
}  // namespace

int main() {
    std::mt19937_64 rng(42);
    std::uniform_real_distribution<double> u(-5.0, 5.0);
    std::vector<slam::Vec3d> pts(30000);
    std::vector<double> ts(pts.size());
    for (size_t i = 0; i < pts.size(); ++i) {
        pts[i] = slam::Vec3d{{u(rng), u(rng), u(rng)}};
        ts[i] = 0.001 * (double) i;
    }
    const slam::GridSamplingOptions o{0.4, 3, 20000};
    int failures = 0;
    try {
        const std::vector<size_t> got = slam::SamplePointsInGrid(pts, o);
        const std::vector<uint64_t> ref = Oracle(pts, o);
        if (got.size() != ref.size()) ++failures;
        for (size_t k = 0; k < got.size() && k < ref.size(); ++k) failures += got[k] != ref[k];
        slam::WorldCloud wc(o);
        const size_t cut[4] = {0, 1000, 1000, pts.size()};   // the second add is empty
        for (int c = 0; c < 3; ++c)
            wc.AddWorldPoints(std::vector<slam::Vec3d>(pts.begin() + cut[c], pts.begin() + cut[c + 1]),
                              std::vector<double>(ts.begin() + cut[c], ts.begin() + cut[c + 1]));
        std::vector<size_t> src;
        const std::vector<slam::WPoint3D> cloud = wc.Points(&src);
        if (cloud.size() != ref.size() || src.size() != ref.size()) ++failures;
        for (size_t k = 0; k < cloud.size() && k < ref.size(); ++k) {
            failures += src[k] != ref[k];
            for (int a = 0; a < 3; ++a) failures += cloud[k].world_point[a] != pts[ref[k]][a];
            failures += cloud[k].raw_point.timestamp != ts[ref[k]];
        }
    } catch (const ct_icp::CticpFailure &e) {
        std::printf("%s\n", e.what());
        std::exit(e.code == CTICP_ERR_NO_DEVICE ? 42 : 1);
    }
    if (failures) {
        std::printf("%d mismatches\n", failures);
        return 1;
    }
    std::printf("WORLD CLOUD FACADE OK\n");
    return 0;
}
