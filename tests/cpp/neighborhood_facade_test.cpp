// slam::TNeighborhood of the C++ facade (ct_icp_b200/odometry.hpp): the three cases of the reference's
// test/unit/SlamCore/test_neighborhood.cxx written against the facade (Vec3d for Eigen::Vector3d, Random() for
// Eigen::Vector3d::Random()), and a batched search and describe against the CPU restatement (tests/oracle_neighborhood).
// Exit 0 and "NEIGHBORHOOD FACADE OK" on success; exit 42 when no device is usable (CTICP_ERR_NO_DEVICE); 1 on a mismatch.
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <random>
#include <vector>

#include "ct_icp_b200/odometry.hpp"

extern "C" void orn_search(const double *, size_t, const double *, size_t, int, double, uint64_t *, double *, int32_t *);
extern "C" void orn_describe(const double *, size_t, const double *, int, double, double, int,
                             cticp_neighborhood_description *);

namespace {
int failures = 0;
void expect(bool ok, const char *what) {
    if (!ok) {
        std::printf("MISMATCH %s\n", what);
        ++failures;
    }
}
std::mt19937_64 rng(42);
slam::Vec3d Random() {   // Eigen::Vector3d::Random(): uniform in [-1, 1]^3
    std::uniform_real_distribution<double> u(-1.0, 1.0);
    return slam::Vec3d{{u(rng), u(rng), u(rng)}};
}

void CaseEigen() {   // TEST(test_neighborhood, eigen)
    int n = 1000;
    std::vector<slam::Vec3d> points;
    points.resize(n);
    for (auto &point : points) point = Random();
    slam::Neighborhood neighborhood(points);
    neighborhood.ComputeNeighborhood(slam::ALL);
    slam::NearestNeighborSearchResult result(10, 0.1);
    neighborhood.SearchNearestNeighbors(Random(), result.ResultSet());
    auto indices = result.Indices();
    expect(indices.size() >= 1, "eigen: indices.size() >= 1");
}

void CaseWorldPoint() {   // TEST(test_neighborhood, world_point)
    int n = 1000;
    std::vector<slam::WPoint3D> points;
    points.resize(n);
    for (auto &point : points) point.WorldPoint() = Random();
    slam::WorldPointNeighborhood neighborhood(points);
    neighborhood.ComputeNeighborhood(slam::ALL);
    slam::NearestNeighborSearchResult result(10, 0.1);
    neighborhood.SearchNearestNeighbors(Random(), result.ResultSet());
    auto indices = result.Indices();
    expect(indices.size() >= 1, "world_point: indices.size() >= 1");
}

void CaseNormals() {   // TEST(test_neighborhood, normals)
    int n = 10;
    std::vector<slam::Vec3d> points(n);
    for (auto &point : points) {
        point = Random();
        point.z() = 1.;
    }
    slam::TNeighborhood<slam::Vec3d> neighborhood(points);
    neighborhood.ComputeNeighborhood(slam::ALL_BUT_KDTREE);
    auto normal = neighborhood.description.normal;
    double dist = normal.dot(slam::Vec3d{{0, 0, 1}});
    expect(std::abs(dist) == 1., "normals: |normal . z| == 1");
}

void CaseBatched() {   // batched search (exact) and describe (error model) against the restatement
    std::normal_distribution<double> g(0.0, 1.0);
    std::vector<slam::Vec3d> points(20000), queries(500);
    for (auto &p : points) p = slam::Vec3d{{300.0 + 4.0 * g(rng), -50.0 + 2.0 * g(rng), 0.3 * g(rng)}};
    for (size_t i = 0; i < queries.size(); ++i) queries[i] = points[i * 7] - slam::Vec3d{{0.01, 0.0, 0.02}};
    slam::Neighborhood nb(points);
    const int k = 20;
    std::vector<uint64_t> idx, ridx(queries.size() * k);
    std::vector<double> d2, rd2(queries.size() * k);
    std::vector<int32_t> cnt, rcnt(queries.size());
    nb.SearchNearestNeighbors(queries, k, 1.0, idx, d2, cnt);
    orn_search(points[0].v, points.size(), queries[0].v, queries.size(), k, 1.0, ridx.data(), rd2.data(), rcnt.data());
    for (size_t i = 0; i < idx.size(); ++i) expect(idx[i] == ridx[i] && d2[i] == rd2[i], "batched search");
    for (size_t q = 0; q < cnt.size(); ++q) expect(cnt[q] == rcnt[q], "batched counts");
    const auto desc = nb.DescribeNeighborhoods(queries, k);
    std::vector<uint64_t> aidx(queries.size() * k);
    std::vector<double> ad2(queries.size() * k);
    std::vector<int32_t> acnt(queries.size());
    orn_search(points[0].v, points.size(), queries[0].v, queries.size(), k, std::numeric_limits<double>::max(),
               aidx.data(), ad2.data(), acnt.data());
    for (size_t q = 0; q < queries.size(); ++q) {
        std::vector<double> nbh;
        for (int j = 0; j < acnt[q]; ++j)
            for (int a = 0; a < 3; ++a) nbh.push_back(points[aidx[q * k + j]][a]);
        cticp_neighborhood_description ref{};
        orn_describe(nbh.data(), (size_t) acnt[q], queries[q].v, CTICP_NB_ALL, 0.8, 0.8, 1, &ref);
        const cticp_neighborhood_description &d = desc[q];
        expect(d.is_valid == ref.is_valid, "describe: is_valid");
        expect(std::abs(d.planarity - ref.planarity) < 1e-9 && std::abs(d.linearity - ref.linearity) < 1e-9,
               "describe: planarity / linearity");
        const double c = std::abs(d.normal[0] * ref.normal[0] + d.normal[1] * ref.normal[1] + d.normal[2] * ref.normal[2]);
        expect(c > 1 - 1e-9, "describe: normal");
        for (int a = 0; a < 3; ++a) expect(std::abs(d.barycenter[a] - ref.barycenter[a]) < 1e-9, "describe: barycenter");
        if (std::abs(ref.planarity - 0.8) > 1e-8 && std::abs(ref.linearity - 0.8) > 1e-8)
            expect(d.type == ref.type, "describe: type");
    }
    nb.ComputeNeighborhood(slam::ALL);   // the set's own description and the reference's classification order
    nb.ClassifyNeighborhood();
    cticp_neighborhood_description ref{};
    orn_describe(points[0].v, points.size(), nullptr, CTICP_NB_ALL, 0.8, 0.8, 1, &ref);
    expect(std::abs(nb.description.planarity - ref.planarity) < 1e-9, "set: planarity");
    expect((int) nb.neighborhood == ref.type, "set: ClassifyNeighborhood");
}
}  // namespace

int main() {
    try {
        CaseEigen();
        CaseWorldPoint();
        CaseNormals();
        CaseBatched();
    } catch (const ct_icp::CticpFailure &e) {
        std::printf("%s\n", e.what());
        std::exit(e.code == CTICP_ERR_NO_DEVICE ? 42 : 1);
    }
    if (failures) {
        std::printf("%d mismatches\n", failures);
        return 1;
    }
    std::printf("NEIGHBORHOOD FACADE OK\n");
    return 0;
}
