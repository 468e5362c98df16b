// Host build of the robust ladder's decision (csrc/frame_policy.h robust_attempt_decide, evaluated by k_frame_policy and
// by the host tail) against a restatement of the reference's control flow: AssessRegistration (odometry.cpp:604-684),
// the acceptance rule and failure counter of RobustRegistration (:780-852) and UpdateMap's robust branch (:855-953).
// Every threshold is put just below, at and just above the value it is compared with; ICP failure flags 0, 1, 4 (and 2,
// the error the host raises); first, middle and last attempts for robust_num_attempts 0, 1, 3, 10; 0..7 consecutive
// failures; robust_minimal_level 0 and 2; the insert overrides; room_for below and above the frame's point count.
#include <cmath>
#include <cstdio>
#include <string>
#include <vector>

#include "frame_policy.h"

using namespace cticp;

namespace model {   // the reference, statement by statement, on a summary whose metrics are given

struct Options {
    double distance_error_threshold, orientation_error_threshold;
    double robust_threshold_relative_orientation, robust_threshold_ego_orientation, robust_relative_trans_threshold;
    int robust_num_attempts, robust_num_attempts_when_rotation, robust_minimal_level;
    bool do_no_insert, always_insert;
};
struct Summary {
    double relative_distance, relative_orientation, ego_orientation;
    bool success;
    int robust_level = 0;   // never copied from the attempt (the reference's quirk): stays 0
    int number_of_attempts;
    std::string error_message;
};
bool AssessRegistration(const Options &o, Summary &s) {
    if (s.relative_distance > o.distance_error_threshold) return false;
    if (s.relative_orientation > o.orientation_error_threshold || s.ego_orientation > o.orientation_error_threshold)
        return false;
    bool success = s.success;
    if (s.robust_level == 0 && (s.relative_orientation > o.robust_threshold_relative_orientation ||
                                s.ego_orientation > o.robust_threshold_ego_orientation)) {
        if (s.robust_level < o.robust_num_attempts_when_rotation) {
            s.error_message = "rotation";
            return false;
        }
    }
    if (s.relative_distance > o.robust_relative_trans_threshold) {
        s.error_message = "translation";
        return false;
    }
    return success;
}
struct Outcome {
    bool assess, accepted;
    int consecutive_failures;   // after the frame (accepted attempts)
    bool points_added, add_points;
    int next_robust_level;
};
// attempt `a` (0-based) of the ladder, summary.number_of_attempts == a before it; consecutive failures before the frame
Outcome Attempt(const Options &o, Summary &s, int cf) {
    Outcome r{};
    bool good = AssessRegistration(o, s);
    r.assess = good;
    s.number_of_attempts++;
    if (!good) {
        if (s.number_of_attempts < o.robust_num_attempts) {
            r.accepted = false;
            return r;
        }
        good = true;
    }
    r.accepted = true;
    cf = s.number_of_attempts > o.robust_num_attempts ? cf + 1 : 0;
    r.consecutive_failures = cf;
    // UpdateMap
    bool add_points = true;
    const bool suspect = s.number_of_attempts >= o.robust_num_attempts;
    if (s.ego_orientation > o.robust_threshold_ego_orientation || s.relative_orientation > o.robust_threshold_relative_orientation)
        add_points = false;
    if (suspect) add_points |= (cf > 5);
    int next = add_points ? o.robust_minimal_level : o.robust_minimal_level + 1;
    if (!s.success)
        next = o.robust_minimal_level + 2;
    else {
        if (s.relative_orientation > o.robust_threshold_relative_orientation || s.ego_orientation > o.robust_threshold_ego_orientation)
            next = o.robust_minimal_level + 1;
        if (s.number_of_attempts > 1) next = o.robust_minimal_level + 1;
    }
    r.points_added = add_points;
    if (o.do_no_insert) add_points = false;
    if (o.always_insert) add_points = true;
    r.add_points = add_points;
    r.next_robust_level = next;
    return r;
}

// slam::AngularDistance on rotation matrices built from the quaternions independently of se3.cuh
double AngularDistance(const double *a, const double *b) {
    auto R = [](const double *q, double m[3][3]) {
        const double n = std::sqrt(q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3]);
        const double x = q[0] / n, y = q[1] / n, z = q[2] / n, w = q[3] / n;
        m[0][0] = 1 - 2 * (y * y + z * z); m[0][1] = 2 * (x * y - z * w);     m[0][2] = 2 * (x * z + y * w);
        m[1][0] = 2 * (x * y + z * w);     m[1][1] = 1 - 2 * (x * x + z * z); m[1][2] = 2 * (y * z - x * w);
        m[2][0] = 2 * (x * z - y * w);     m[2][1] = 2 * (y * z + x * w);     m[2][2] = 1 - 2 * (x * x + y * y);
    };
    double A[3][3], B[3][3], tr = 0;
    R(a, A);
    R(b, B);
    for (int i = 0; i < 3; ++i)
        for (int k = 0; k < 3; ++k) tr += A[i][k] * B[i][k];   // trace(A · Bᵀ)
    const double n = std::fmax(std::fmin((tr - 1) / 2, 1.0), -1.0);
    return std::acos(n) * 180.0 / M_PI;
}

}  // namespace model

struct Poses {
    double qb[4], qe[4], tb[3], te[3], prev_qe[4], prev_te[3];
};

static void axis_angle(double ax, double ay, double az, double deg, double *q) {
    const double n = std::sqrt(ax * ax + ay * ay + az * az), h = 0.5 * deg * M_PI / 180.0;
    q[0] = std::sin(h) * ax / n; q[1] = std::sin(h) * ay / n; q[2] = std::sin(h) * az / n; q[3] = std::cos(h);
}

// just below, at and just above each value the threshold is compared with
static std::vector<double> levels(std::initializer_list<double> values) {
    std::vector<double> out;
    for (double v : values) {
        out.push_back(std::nextafter(v, -INFINITY));
        out.push_back(v);
        out.push_back(std::nextafter(v, INFINITY));
    }
    return out;
}

// first, middle and last attempt of a ladder of robust_num_attempts = N (a ladder runs at least one attempt)
static std::vector<int> attempts_of(int N) {
    std::vector<int> out{0};
    if (N / 2 > 0 && N / 2 < N - 1) out.push_back(N / 2);
    if (N - 1 > 0) out.push_back(N - 1);
    return out;
}

int main() {
    std::vector<Poses> scenes;
    {   // small, moderate and large motions; begin / end / previous rotations about different axes
        const double degs[][3] = {{0.3, 0.5, 0.2}, {4.0, 2.5, 6.0}, {15.0, 40.0, 1.0}};
        const double trans[][2] = {{0.02, 0.05}, {0.8, 1.3}, {3.0, 0.4}};
        for (int i = 0; i < 3; ++i) {
            Poses p;
            axis_angle(0.1, 0.2, 1.0, degs[i][0], p.qb);
            axis_angle(0.3, -0.1, 1.0, degs[i][0] + degs[i][1], p.qe);
            axis_angle(-0.2, 0.4, 1.0, degs[i][2], p.prev_qe);
            p.tb[0] = 10.0; p.tb[1] = -3.0; p.tb[2] = 0.5;
            p.te[0] = 10.0 + trans[i][0]; p.te[1] = -3.0 + 0.5 * trans[i][0]; p.te[2] = 0.5;
            p.prev_te[0] = 10.0 - trans[i][1]; p.prev_te[1] = -3.0; p.prev_te[2] = 0.4;
            scenes.push_back(p);
        }
    }
    long cases = 0, bad = 0;
    double worst_metric = 0;
    for (const Poses &p : scenes) {
        const Q4 qb{p.qb[0], p.qb[1], p.qb[2], p.qb[3]}, qe{p.qe[0], p.qe[1], p.qe[2], p.qe[3]};
        const V3 tb{p.tb[0], p.tb[1], p.tb[2]}, te{p.te[0], p.te[1], p.te[2]};
        FramePolicyIn in{};
        RobustPolicyIn r{};
        for (int i = 0; i < 4; ++i) r.prev_qe[i] = p.prev_qe[i];
        for (int i = 0; i < 3; ++i) r.prev_te[i] = p.prev_te[i];
        r.enabled = 1;
        // the metrics, against independent definitions (RobustRegistration :802-821)
        const RobustDecision m = robust_attempt_decide(qb, tb, qe, te, 0, 100, in, r);
        const double dc = std::sqrt(std::pow(p.tb[0] - p.prev_te[0], 2) + std::pow(p.tb[1] - p.prev_te[1], 2) + std::pow(p.tb[2] - p.prev_te[2], 2));
        const double rd = std::sqrt(std::pow(p.te[0] - p.tb[0], 2) + std::pow(p.te[1] - p.tb[1], 2) + std::pow(p.te[2] - p.tb[2], 2));
        const double ro = model::AngularDistance(p.prev_qe, p.qe), eg = model::AngularDistance(p.qb, p.qe);
        for (double e : {std::fabs(m.distance_correction - dc), std::fabs(m.relative_distance - rd),
                         std::fabs(m.relative_orientation - ro), std::fabs(m.ego_orientation - eg)})
            worst_metric = std::fmax(worst_metric, e);
        // thresholds against the function's own metrics (so that "at" is exactly at)
        const std::vector<double> L_dist = levels({m.relative_distance}), L_orient = levels({m.relative_orientation, m.ego_orientation}),
                                  L_rel = levels({m.relative_orientation}), L_ego = levels({m.ego_orientation}),
                                  L_trans = levels({m.relative_distance});
        for (double t_dist : L_dist)
        for (double t_orient : L_orient)
        for (double t_rel : L_rel)
        for (double t_ego : L_ego)
        for (double t_trans : L_trans)
        for (int when_rotation : {0, 2})
        for (int failed : {0, 1, 4, 2})
        for (int N : {0, 1, 3, 10})
        for (int a : attempts_of(N)) {
            for (int cf = 0; cf <= 7; ++cf)
            for (int minimal : {0, 2})
            for (int ov = 0; ov < 4; ++ov)
            for (int room : {50, 150}) {
                model::Options o{t_dist, t_orient, t_rel, t_ego, t_trans, N, when_rotation, minimal, (ov & 1) != 0, (ov & 2) != 0};
                model::Summary s{m.relative_distance, m.relative_orientation, m.ego_orientation, failed == 0, 0, a, ""};
                const model::Outcome want = model::Attempt(o, s, cf);
                in.distance_error_threshold = t_dist;
                in.orientation_error_threshold = t_orient;
                in.do_no_insert = o.do_no_insert;
                in.always_insert = o.always_insert;
                in.room_for = room;
                r.threshold_relative_orientation = t_rel;
                r.threshold_ego_orientation = t_ego;
                r.relative_trans_threshold = t_trans;
                r.num_attempts_when_rotation = when_rotation;
                r.minimal_level = minimal;
                r.number_of_attempts = a + 1;
                r.last_attempt = a + 1 >= N;
                r.consecutive_failures = a + 1 > N ? cf + 1 : 0;
                const RobustDecision d = robust_attempt_decide(qb, tb, qe, te, failed, 100, in, r);
                ++cases;
                const std::string msg = d.reject_reason == kRejectRotation ? "rotation"
                                        : d.reject_reason == kRejectTranslation ? "translation" : "";
                bool ok = d.assess_ok == (int) want.assess && d.accepted == (int) want.accepted && msg == s.error_message;
                int want_action;
                if (failed == 2) want_action = kFrameSkip;
                else if (!want.accepted) want_action = kFrameRetry;
                else if (want.add_points && 100 > room) want_action = kFrameDeferred;
                else want_action = want.add_points ? kFrameInsert : kFrameEvict;
                ok = ok && d.action == want_action;
                if (want.accepted)
                    ok = ok && d.add_points_policy == (int) want.points_added && d.add_points == (int) want.add_points &&
                         d.next_robust_level == want.next_robust_level && r.consecutive_failures == want.consecutive_failures;
                if (!ok) {
                    if (bad < 10)
                        printf("mismatch: thr %.17g %.17g %.17g %.17g %.17g rot %d failed %d N %d a %d cf %d min %d ov %d room %d: "
                               "assess %d/%d accepted %d/%d action %d/%d add %d/%d next %d/%d msg '%s'/'%s'\n",
                               t_dist, t_orient, t_rel, t_ego, t_trans, when_rotation, failed, N, a, cf, minimal, ov, room,
                               d.assess_ok, want.assess, d.accepted, want.accepted, d.action, want_action, d.add_points,
                               want.add_points, d.next_robust_level, want.next_robust_level, msg.c_str(), s.error_message.c_str());
                    ++bad;
                }
            }
        }
    }
    if (!(worst_metric < 1e-9)) { printf("metrics differ from their definitions by %.3e\n", worst_metric); ++bad; }
    if (bad) { printf("FAILED: %ld of %ld\n", bad, cases); return 1; }
    printf("ROBUST POLICY OK (%ld cases, metrics within %.1e)\n", cases, worst_metric);
    return 0;
}
