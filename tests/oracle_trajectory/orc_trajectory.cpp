// ORACLE — TEST INFRASTRUCTURE ONLY. The cticp_trajectory_* entry points of include/cticp.h, prefixed orc_, over
// orc_trajectory.h: the tests drive the engine and this restatement through the same Python binding. Host memory only.
// Built by __graft_entry__.build() and by tests/oracle_trajectory_lib.py into liborc_trajectory.so.
#include <cstring>
#include <memory>
#include <string>
#include <vector>

#include "../../include/cticp.h"
#include "orc_trajectory.h"

namespace {
thread_local std::string g_last_error;

template <typename F>
int Guard(F &&f) {
    try {
        return f();
    } catch (const std::invalid_argument &e) {
        g_last_error = e.what();
        return CTICP_ERR_INVALID_ARGUMENT;
    } catch (const std::exception &e) {
        g_last_error = e.what();
        return CTICP_ERR_INTERNAL;
    }
}

orc::Pose FromC(const cticp_pose &c) {
    orc::Pose p;
    p.pose.quat = orc::Quat(c.quat[0], c.quat[1], c.quat[2], c.quat[3]);   // as given: no normalisation
    p.pose.tr = orc::Vec3(c.tr[0], c.tr[1], c.tr[2]);
    p.ref_timestamp = c.ref_timestamp;
    p.dest_timestamp = c.dest_timestamp;
    p.ref_frame_id = c.ref_frame_id;
    p.dest_frame_id = c.dest_frame_id;
    return p;
}
cticp_pose ToC(const orc::Pose &p) {
    cticp_pose c;
    c.quat[0] = p.pose.quat.x; c.quat[1] = p.pose.quat.y; c.quat[2] = p.pose.quat.z; c.quat[3] = p.pose.quat.w;
    c.tr[0] = p.pose.tr.x; c.tr[1] = p.pose.tr.y; c.tr[2] = p.pose.tr.z;
    c.ref_timestamp = p.ref_timestamp;
    c.dest_timestamp = p.dest_timestamp;
    c.ref_frame_id = p.ref_frame_id;
    c.dest_frame_id = p.dest_frame_id;
    return c;
}

// static_cast<double> of one scalar of a record
double Scalar(const unsigned char *p, int dtype) {
    switch (dtype) {
        case CTICP_DTYPE_INT8: { int8_t v; memcpy(&v, p, 1); return v; }
        case CTICP_DTYPE_UINT8: { uint8_t v; memcpy(&v, p, 1); return v; }
        case CTICP_DTYPE_INT16: { int16_t v; memcpy(&v, p, 2); return v; }
        case CTICP_DTYPE_UINT16: { uint16_t v; memcpy(&v, p, 2); return v; }
        case CTICP_DTYPE_INT32: { int32_t v; memcpy(&v, p, 4); return v; }
        case CTICP_DTYPE_UINT32: { uint32_t v; memcpy(&v, p, 4); return v; }
        case CTICP_DTYPE_FLOAT32: { float v; memcpy(&v, p, 4); return v; }
        case CTICP_DTYPE_FLOAT64: { double v; memcpy(&v, p, 8); return v; }
        default: throw std::invalid_argument("unknown dtype");
    }
}
size_t DtypeSize(int dtype) {
    static const size_t kSize[9] = {0, 1, 1, 2, 2, 4, 4, 4, 8};
    return dtype >= 1 && dtype <= 8 ? kSize[dtype] : 0;
}
}  // namespace

struct orc_trajectory {
    orc::LinearContinuousTrajectory t;
};

extern "C" {

const char *orc_last_error(void) { return g_last_error.c_str(); }

int orc_trajectory_create(const cticp_pose *poses, size_t n, int device, orc_trajectory **out) {
    (void) device;
    return Guard([&] {
        if (!poses || !out) throw std::invalid_argument("null argument");
        std::vector<orc::Pose> v;
        for (size_t i = 0; i < n; ++i) v.push_back(FromC(poses[i]));
        *out = new orc_trajectory{orc::LinearContinuousTrajectory::Create(std::move(v))};
        return 0;
    });
}
void orc_trajectory_destroy(orc_trajectory *t) { delete t; }
int64_t orc_trajectory_poses(orc_trajectory *t, cticp_pose *dst, size_t cap) {
    const auto &p = t->t.Poses();
    for (size_t i = 0; i < p.size() && i < cap && dst; ++i) dst[i] = ToC(p[i]);
    return (int64_t) p.size();
}
int orc_trajectory_interpolate(orc_trajectory *t, const double *timestamps, const uint32_t *frame_ids, size_t m,
                               cticp_pose *out) {
    return Guard([&] {
        std::vector<cticp_pose> r(m);
        for (size_t i = 0; i < m; ++i)
            r[i] = ToC(frame_ids ? t->t.InterpolatePoseWithFrameId(timestamps[i], frame_ids[i])
                                 : t->t.InterpolatePose(timestamps[i]));
        if (m) memcpy(out, r.data(), sizeof(cticp_pose) * m);
        return 0;
    });
}
// test tap: GetClosestPosesIds(t[, frame_id], clip_on_bounds = true); frame_id < 0: the overload without one
int orc_trajectory_closest_ids(orc_trajectory *t, double timestamp, int64_t frame_id, uint64_t *lo, uint64_t *up) {
    return Guard([&] {
        size_t l = 0, u = 0;
        if (frame_id < 0) t->t.GetClosestPosesIds(timestamp, l, u);
        else t->t.GetClosestPosesIds(timestamp, (uint32_t) frame_id, l, u);
        *lo = l;
        *up = u;
        return 0;
    });
}
// RawPointsToWorldPoints (src/SlamCore/pointcloud.cxx:313-326) point by point; the records are written only once every
// point has been transformed
int64_t orc_trajectory_transform(orc_trajectory *t, const cticp_cloud_view *c, const uint64_t *segment_ends,
                                 const uint32_t *segment_frame_ids, size_t num_segments, const cticp_cloud_sink *sink) {
    int64_t count = 0;
    int rc = Guard([&] {
        if (!c || !sink || !sink->world) throw std::invalid_argument("bad argument");
        const size_t n = c->num_points, xs = c->xyz_dtype == CTICP_DTYPE_FLOAT32 ? 4 : 8;
        if (!DtypeSize(c->t_dtype)) throw std::invalid_argument("unknown timestamp dtype");
        if (num_segments && segment_ends[num_segments - 1] != n) throw std::invalid_argument("segments");
        const size_t m = std::min<size_t>(sink->capacity_points, n);
        std::vector<orc::Vec3> w(m);
        std::vector<double> ts(m);
        size_t seg = 0;
        for (size_t i = 0; i < m; ++i) {
            const auto *rec = static_cast<const unsigned char *>(c->data) + i * c->point_step;
            const orc::Vec3 raw(Scalar(rec + c->xyz_offset, c->xyz_dtype), Scalar(rec + c->xyz_offset + xs, c->xyz_dtype),
                                Scalar(rec + c->xyz_offset + 2 * xs, c->xyz_dtype));
            ts[i] = Scalar(rec + c->t_offset, c->t_dtype);
            if (num_segments) {
                while (segment_ends[seg] <= i) ++seg;
                w[i] = t->t.TransformPoint(raw, ts[i], segment_frame_ids[seg]);
            } else {
                w[i] = t->t.TransformPoint(raw, ts[i]);
            }
        }
        for (size_t i = 0; i < m; ++i) {
            auto *rec = static_cast<unsigned char *>(sink->data) + i * sink->point_step;
            if (sink->xyz_dtype == CTICP_DTYPE_FLOAT32) {
                const float v[3] = {(float) w[i].x, (float) w[i].y, (float) w[i].z};
                memcpy(rec + sink->xyz_offset, v, sizeof(v));
            } else {
                const double v[3] = {w[i].x, w[i].y, w[i].z};
                memcpy(rec + sink->xyz_offset, v, sizeof(v));
            }
            if (sink->t_dtype == CTICP_DTYPE_FLOAT32) {
                const float v = (float) ts[i];
                memcpy(rec + sink->t_offset, &v, 4);
            } else if (sink->t_dtype == CTICP_DTYPE_FLOAT64) {
                memcpy(rec + sink->t_offset, &ts[i], 8);
            }
        }
        count = (int64_t) n;
        return 0;
    });
    return rc < 0 ? rc : count;
}

}  // extern "C"
