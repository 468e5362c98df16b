// orc_grid.cpp — a plain C++ restatement of slam::SamplePointsInGrid (include/SlamCore/algorithm/grid_sampling.h:48-79)
// and slam::Voxel::Coordinates (src/SlamCore/types.cxx:13-20), written from their documented behaviour, with the order
// the engine promises: voxels in order of first appearance, each voxel's points in input order. It exports the engine's
// cticp_sample_points_in_grid signature under the prefix orc_, so the tests drive both through the same binding.
// TEST INFRASTRUCTURE.
#include <cmath>
#include <cstdint>
#include <cstring>
#include <unordered_map>
#include <vector>

#include "../../include/cticp.h"

namespace {

struct Key {
    int x, y, z;
    bool operator==(const Key &o) const { return x == o.x && y == o.y && z == o.z; }
};
struct KeyHash {
    size_t operator()(const Key &k) const {
        return (size_t) k.x * 73856093u ^ (size_t) k.y * 19349663u ^ (size_t) k.z * 83492791u;
    }
};

// Voxel::Coordinates: int(p / grid_size) per axis; false where the engine rejects the point (non-finite, or a voxel
// coordinate outside [-2^20, 2^20): the reference's int() of such a value is undefined)
bool Coordinates(const double *p, double grid, Key &k) {
    int v[3];
    for (int a = 0; a < 3; ++a) {
        const double q = p[a] / grid;
        if (!(std::fabs(q) < 2097152.0)) return false;
        v[a] = int(q);
        if (v[a] < -(1 << 20) || v[a] >= (1 << 20)) return false;
    }
    k = Key{v[0], v[1], v[2]};
    return true;
}

}  // namespace

extern "C" {

const char *orc_last_error(void) { return "oracle: invalid argument"; }

void orc_default_grid_sampling_options(cticp_grid_sampling_options *out) {
    std::memset(out, 0, sizeof(*out));
    out->grid_size = 1.0;
    out->num_points_per_voxel = 1;
    out->max_num_points = -1;
}

int64_t orc_sample_points_in_grid(int, const cticp_grid_sampling_options *o, const double *xyz, size_t stride_bytes,
                                  size_t n, uint64_t *out_indices, size_t cap) {
    if (!o || !(std::isfinite(o->grid_size) && o->grid_size > 0.0)) return CTICP_ERR_INVALID_ARGUMENT;
    if (o->num_points_per_voxel < 0 || o->num_points_per_voxel > 64) return CTICP_ERR_UNSUPPORTED;
    std::unordered_map<Key, size_t, KeyHash> id;          // voxel → its rank of first appearance
    std::vector<std::vector<uint64_t>> voxels;
    for (size_t i = 0; i < n; ++i) {
        const double *p = reinterpret_cast<const double *>(reinterpret_cast<const char *>(xyz) + stride_bytes * i);
        Key k;
        if (!Coordinates(p, o->grid_size, k)) continue;
        auto it = id.find(k);
        if (it == id.end()) {                              // the first point of a voxel is always kept
            id.emplace(k, voxels.size());
            voxels.push_back({(uint64_t) i});
        } else if (voxels[it->second].size() < (size_t) o->num_points_per_voxel) {
            voxels[it->second].push_back(i);
        }
    }
    const size_t limit = o->max_num_points < 0 ? SIZE_MAX : (size_t) o->max_num_points;
    std::vector<uint64_t> out;
    for (const auto &v : voxels) {                        // size() > limit is tested before each push
        for (uint64_t i : v) {
            if (out.size() > limit) break;
            out.push_back(i);
        }
        if (out.size() > limit) break;
    }
    for (size_t j = 0; j < out.size() && j < cap && out_indices; ++j) out_indices[j] = out[j];
    return (int64_t) out.size();
}

}  // extern "C"
