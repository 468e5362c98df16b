// The dataset readers of the C++ facade (ct_icp_b200/odometry.hpp) over the C ABI: ReadPLYLayout and LoadGroundTruth on
// the host, then an NCLT stream of three packets decoded and the KITTI filter applied on the device.
// Exit 0 and "DATASET FACADE OK" on success; exit 42 when no device is usable (CTICP_ERR_NO_DEVICE); 1 on a mismatch.
#include <cmath>
#include <cstdio>
#include <cstring>
#include <string>
#include <vector>

#include "ct_icp_b200/odometry.hpp"

static int fail(const char *what) {
    std::printf("MISMATCH: %s\n", what);
    return 1;
}

static void put(std::vector<unsigned char> &b, const void *p, size_t n) {
    const unsigned char *c = static_cast<const unsigned char *>(p);
    b.insert(b.end(), c, c + n);
}

// one packet: 4 x u16 44444, u32 num_hits, u64 utime, u32 pad, then the hits (u16 x y z, u8 intensity, u8 laser)
static void packet(std::vector<unsigned char> &b, uint64_t utime, const std::vector<std::array<uint16_t, 3>> &hits) {
    const uint16_t magic[4] = {44444, 44444, 44444, 44444};
    const uint32_t n = (uint32_t) hits.size(), pad = 0;
    put(b, magic, 8);
    put(b, &n, 4);
    put(b, &utime, 8);
    put(b, &pad, 4);
    for (const auto &h : hits) {
        put(b, h.data(), 6);
        const unsigned char il[2] = {7, 3};
        put(b, il, 2);
    }
}

int main() {
    const std::string ply = "ply\nformat binary_little_endian 1.0\nelement vertex 2\nproperty float x\nproperty float y\n"
                            "property float z\nproperty double timestamp\nend_header\n";
    std::vector<unsigned char> file(ply.begin(), ply.end());
    file.resize(file.size() + 2 * 20);
    const cticp_ply_layout lay = ct_icp::ReadPLYLayout(file.data(), file.size());
    if (lay.num_points != 2 || lay.point_step != 20 || lay.xyz_dtype != CTICP_DTYPE_FLOAT32 ||
        lay.t_dtype != CTICP_DTYPE_FLOAT64 || lay.t_offset != 12 || lay.body_offset != ply.size())
        return fail("ReadPLYLayout");
    const std::vector<slam::Pose> gt = ct_icp::LoadGroundTruth(CTICP_DATASET_KITTI_CARLA,
                                                               "1 0 0 1 0 1 0 2 0 0 1 3\n\n1 0 0 4 0 1 0 5 0 0 1 6\n");
    if (gt.size() != 2 || gt[1].pose.tr.v[0] != 4 || gt[1].dest_frame_id != 1 || gt[1].dest_timestamp != 0.1)
        return fail("LoadGroundTruth");
    try {
        std::vector<unsigned char> bytes;
        packet(bytes, 1000, {{{20000, 20000, 20000}}, {{20200, 19800, 21000}}});
        packet(bytes, 1001, {});
        packet(bytes, 1002, {{{0, 65535, 1}}});
        ct_icp::NCLTHits hits(bytes.data(), bytes.size(), 2, true, 0);
        if (hits.NumFrames() != 2 || hits.NumPackets() != 3 || hits.NumHits() != 3 || hits.BytesUsed() != bytes.size())
            return fail("NCLTHits counts");
        std::vector<uint64_t> ends;
        std::vector<slam::WPoint3D> pts = hits.ReadFrames(0, 2, &ends);
        if (pts.size() != 3 || ends[0] != 2 || ends[1] != 3) return fail("ReadFrames ends");
        if (pts[1].RawPoint()[0] != 20200 * 0.005 - 100.0 || pts[2].RawPoint()[1] != 65535 * 0.005 - 100.0 ||
            pts[2].Timestamp() != 1002.0 || pts[2].index_frame != 1)
            return fail("ReadFrames values");
        const auto info = hits.FrameInfo(0, 2);
        if (info[0].num_points != 2 || info[0].t_first != 1000.0 || info[1].t_max != 1002.0) return fail("FrameInfo");
        std::vector<slam::WPoint3D> f(2);
        f[0].RawPoint() = slam::Vec3d{{10.0, 3.0, 1.0}};
        f[1].RawPoint() = slam::Vec3d{{10.0, 3.0, -6.0}};
        const double n0 = f[0].RawPoint().norm();
        ct_icp::KittiFrameFilter(f, 0);
        if (std::fabs(f[0].RawPoint().norm() - n0) > 1e-12 * n0 || f[0].RawPoint()[2] <= 1.0 ||
            f[1].RawPoint().norm() != 0.0)
            return fail("KittiFrameFilter");
    } catch (const ct_icp::CticpFailure &e) {
        std::printf("%s\n", e.what());
        return e.code == CTICP_ERR_NO_DEVICE ? 42 : 1;
    }
    std::printf("DATASET FACADE OK\n");
    return 0;
}
