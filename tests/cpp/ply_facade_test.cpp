// The PLY writers and the pose reader of the C++ facade (ct_icp_b200/odometry.hpp) over the C ABI. argv[1] is a
// directory: five WPoint3D records go to default.ply (WritePLY's default mapper), float.ply and double.ply, and three
// poses to poses.ply, which ReadPosesFromPLY must read back exactly.
// Exit 0 and "PLY FACADE OK" on success; exit 42 when no device is usable (CTICP_ERR_NO_DEVICE); 1 on a mismatch.
#include <cstdio>
#include <cstring>
#include <fstream>
#include <sstream>
#include <string>
#include <vector>

#include "ct_icp_b200/odometry.hpp"

static int fail(const char *what) {
    std::printf("MISMATCH: %s\n", what);
    return 1;
}

int main(int argc, char **argv) {
    const std::string dir = argc > 1 ? argv[1] : ".";
    std::vector<slam::WPoint3D> points(5);
    for (int i = 0; i < 5; ++i) {   // tests/test_ply_facade.py rebuilds these records
        points[i].RawPoint() = slam::Vec3d{{1.5 * i, -1.0 * i, 0.25 * i}};
        points[i].Timestamp() = 0.1 * i;
        points[i].WorldPoint() = slam::Vec3d{{1.5 * i + 10.0, -1.0 * i + 10.0, 0.25 * i + 10.0}};
        points[i].index_frame = 7u * (unsigned) i;
    }
    std::vector<slam::Pose> poses(3);
    for (int i = 0; i < 3; ++i) {
        poses[i].pose.quat = slam::Quatd{{0.1 * i, 0.2, -0.3, 0.9}};
        poses[i].pose.tr = slam::Vec3d{{1.0 * i, 2.0, 3.0}};
        poses[i].ref_timestamp = 0.5 * i;
        poses[i].dest_timestamp = 0.5 * i + 0.1;
        poses[i].ref_frame_id = (slam::frame_id_t) i;
        poses[i].dest_frame_id = (slam::frame_id_t) -1;
    }
    try {
        slam::WritePLY(dir + "/default.ply", points);
        slam::WritePLY(dir + "/float.ply", points, slam::WPoint3DFloatSchema());
        slam::WritePLY(dir + "/double.ply", points, slam::WPoint3DDoubleSchema());
        slam::SavePosesAsPLY(dir + "/poses.ply", poses);
        std::ostringstream os;
        slam::SavePosesAsPLY(os, poses);
        std::istringstream is(os.str());
        const std::vector<slam::Pose> back = slam::ReadPosesFromPLY(is);
        if (back.size() != poses.size()) return fail("ReadPosesFromPLY count");
        for (size_t i = 0; i < poses.size(); ++i)
            if (std::memcmp(back[i].pose.quat.c, poses[i].pose.quat.c, 32) ||
                std::memcmp(back[i].pose.tr.v, poses[i].pose.tr.v, 24) ||
                back[i].ref_timestamp != poses[i].ref_timestamp || back[i].dest_timestamp != poses[i].dest_timestamp ||
                back[i].ref_frame_id != poses[i].ref_frame_id || back[i].dest_frame_id != poses[i].dest_frame_id)
                return fail("ReadPosesFromPLY values");
        if (slam::ReadPosesFromPLY(dir + "/poses.ply").size() != 3) return fail("ReadPosesFromPLY(path)");
    } catch (const ct_icp::CticpFailure &e) {
        std::printf("%s\n", e.what());
        return e.code == CTICP_ERR_NO_DEVICE ? 42 : 1;
    }
    std::printf("PLY FACADE OK\n");
    return 0;
}
