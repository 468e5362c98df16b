// The facade's YAML readers (ct_icp_b200/include/ct_icp_b200/odometry.hpp, ct_icp::yaml_to_*) over the stub node of
// yaml_node_stub.h. usage: config_facade_test odometry|dataset TREE_FILE. Prints "OK <hex bytes of the
// OdometryOptions>" or "OK <the DatasetOptions fields>", or "ERR <message>" when the reader throws.
#include <cstdio>
#include <fstream>

#include "ct_icp_b200/odometry.hpp"
#include "yaml_node_stub.h"

int main(int argc, char **argv) {
    if (argc != 3) return 2;
    std::ifstream is(argv[2], std::ios::binary);
    const yaml_stub::Node node = yaml_stub::Node::Read(is);
    try {
        if (std::string(argv[1]) == "odometry") {
            const ct_icp::OdometryOptions o = ct_icp::yaml_to_odometry_options(node);
            const cticp_odometry_options &c = o;
            const unsigned char *p = reinterpret_cast<const unsigned char *>(&c);
            std::printf("OK ");
            for (size_t i = 0; i < sizeof(cticp_odometry_options); ++i) std::printf("%02x", p[i]);
            std::printf("\n");
        } else {
            const ct_icp::DatasetOptions d = ct_icp::yaml_to_dataset_options_vector(node).at(0);
            std::printf("OK %s|%s|%d|%.17g|%.17g|%d|%d", d.dataset.c_str(), d.root_path.c_str(), (int) d.fail_if_incomplete,
                        d.min_dist_lidar_center, d.max_dist_lidar_center, d.nclt_num_aggregated_pc,
                        (int) d.use_all_datasets);
            for (const auto &s : d.sequence_options)
                std::printf("|%s,%d,%d", s.sequence_name.c_str(), s.start_frame_id, s.max_num_frames);
            std::printf("\n");
        }
    } catch (const std::exception &e) {
        std::printf("ERR %s\n", e.what());
    }
    return 0;
}
