// The snapshot format (csrc/snapshot_format.h) without a GPU: synthetic odometry and map snapshots written with the
// engine's writer helpers round-trip through snap::Validate; truncations, single-bit flips and structural faults that
// carry a valid checksum are refused.
#include <cstdio>
#include <cstdlib>
#include <limits>
#include <random>
#include <vector>

#include "snapshot_format.h"

using namespace cticp;

static int g_failures = 0;
#define CHECK(cond, ...)                                                   \
    do {                                                                   \
        if (!(cond)) {                                                     \
            ++g_failures;                                                  \
            if (g_failures < 20) {                                         \
                fprintf(stderr, "FAIL %s:%d: ", __FILE__, __LINE__);      \
                fprintf(stderr, __VA_ARGS__);                              \
                fprintf(stderr, "\n");                                     \
            }                                                              \
        }                                                                  \
    } while (0)

struct Synthetic {
    std::vector<uint8_t> bytes;
    snap::Layout layout;
    snap::MapMeta meta;
    uint64_t level_payload[CTICP_MAX_RESOLUTIONS];   // offsets in bytes
};

static cticp_map_options MapOptions(int levels, bool normals) {
    cticp_map_options o{};
    o.num_resolutions = levels;
    o.select_valid_normals_direction = normals ? 1 : 0;
    o.max_frames_to_keep = 1;
    o.default_radius = 0.8;
    const int B[3] = {8, 5, 3};
    for (int i = 0; i < levels; ++i) {
        o.resolutions[i].resolution = 0.2 * (i + 1);
        o.resolutions[i].min_distance_between_points = 0.01;
        o.resolutions[i].max_num_points = B[i % 3];
    }
    return o;
}

// A snapshot of `kind` with `levels` levels of 1024 / 2048 slots, a random set of live voxels and tombstones per level
static Synthetic Make(uint32_t kind, int levels, bool normals, uint64_t frames, unsigned seed) {
    std::mt19937_64 rng(seed);
    Synthetic s;
    snap::MapMeta &m = s.meta;
    m.options = MapOptions(levels, normals);
    m.num_levels = (uint32_t) levels;
    m.has_normals = normals ? 1 : 0;
    m.frame_count = frames;
    struct Rec { uint32_t slot, count; uint64_t key; };
    std::vector<std::vector<Rec>> recs(levels);
    for (int i = 0; i < levels; ++i) {
        snap::LevelMeta &L = m.levels[i];
        L.cap = 1024u << (i & 1);
        L.B = (uint32_t) m.options.resolutions[i].max_num_points;
        for (uint32_t slot = 0; slot < L.cap; ++slot) {
            const unsigned r = (unsigned) (rng() % 16);
            if (r < 11) continue;
            Rec rec{slot, 0, 0};
            if (r == 11) {
                rec.key = snap::kKeyTomb;
                ++L.num_tombs;
            } else {
                rec.key = rng() & ((1ull << 63) - 1);
                rec.count = 1 + (uint32_t) (rng() % L.B);
                ++L.num_voxels;
                L.num_points += rec.count;
            }
            recs[i].push_back(rec);
        }
        L.records = recs[i].size();
        L.num_touched = (uint32_t) (rng() % 100);
    }
    uint64_t size[snap::kNumSections] = {};
    cticp_odometry_options o{};
    o.map_options = m.options;
    o.neighborhood_strategy.type = CTICP_STRATEGY_DISTANCE_BASED;
    snap::HostState hs;
    std::vector<cticp_frame> traj;
    if (kind == snap::kKindOdometry) {
        hs.registered_frames = 3 + (int) (rng() % 5);
        hs.next_robust_level = 2;
        hs.cum_distance = 1.25;
        hs.last_num_keypoints = 4321;
        hs.default_model_present = 1;
        for (int k = 0; k < hs.registered_frames; ++k) {
            cticp_frame f{};
            f.begin_pose.quat[3] = 1.0;
            f.end_pose.quat[3] = 1.0;
            f.end_pose.tr[0] = 0.5 * k;
            f.begin_pose.dest_frame_id = f.end_pose.dest_frame_id = (uint32_t) k;
            traj.push_back(f);
        }
        size[snap::kSecOptions] = sizeof(o);
        size[snap::kSecHost] = snap::kHostStateBytes;
        size[snap::kSecTrajectory] = 8 + snap::kFrameBytes * traj.size();
    }
    size[snap::kSecMap] = snap::MapSectionBytes(m);
    size[snap::kSecOrigins] = snap::OriginsBytes(m);
    s.layout = snap::MakeLayout(kind, size);
    s.bytes.assign(s.layout.total, 0xAB);
    uint8_t *out = s.bytes.data();
    snap::WriteHeader(out, s.layout);
    snap::Writer w(out, s.layout.offset[snap::kSecOptions]);
    if (kind == snap::kKindOdometry) {
        w.bytes(&o, sizeof(o));
        snap::WriteHostState(w, hs);
        w.u64(traj.size());
        for (const auto &f : traj) w.frame(f);
    }
    snap::WriteMapHeader(w, m);
    for (int i = 0; i < levels; ++i) {
        s.level_payload[i] = w.off;
        for (const Rec &r : recs[i]) { w.u32(r.slot); w.u32(r.count); w.u64(r.key); }
        for (const Rec &r : recs[i])
            for (uint32_t j = 0; j < r.count; ++j) {
                const float q[4] = {(float) (rng() % 1000) * 1e-3f, 0.25f, -0.125f,
                                    (float) (1 + rng() % (frames ? frames : 1)) * ((rng() & 1) ? 1.f : -1.f)};
                w.bytes(q, 16);
            }
        if (normals)
            for (size_t k = 0; k < recs[i].size(); ++k) { w.f64(0.0); w.f64(0.0); w.f64(1.0); w.f64(1.0); }
    }
    for (uint64_t f = 0; f < 3 * snap::OriginsBytes(m) / 24; ++f) w.f64(0.1 * (double) f);
    CHECK(w.off == s.layout.total, "writer ended at %zu of %llu", w.off, (unsigned long long) s.layout.total);
    snap::Seal(out, s.layout);
    return s;
}

static bool Accepts(const std::vector<uint8_t> &b, uint32_t kind, size_t n) {
    snap::Parsed p;
    std::string why;
    return snap::Validate(b.data(), n, kind, &p, &why);
}
static bool Accepts(const std::vector<uint8_t> &b, uint32_t kind) { return Accepts(b, kind, b.size()); }

static void Reseal(Synthetic &s) { snap::Seal(s.bytes.data(), s.layout); }

// offsets of record k of level i
static size_t RecordAt(const Synthetic &s, int i, uint64_t k) { return s.level_payload[i] + k * snap::kRecordBytes; }
static void Put32(Synthetic &s, size_t at, uint32_t v) { memcpy(s.bytes.data() + at, &v, 4); }
static uint32_t Get32(const Synthetic &s, size_t at) { uint32_t v; memcpy(&v, s.bytes.data() + at, 4); return v; }

static void TestKind(uint32_t kind, int levels, bool normals, unsigned seed) {
    const uint64_t frames = normals ? 37 : 23;
    Synthetic s = Make(kind, levels, normals, frames, seed);
    // round trip
    snap::Parsed p;
    std::string why;
    CHECK(snap::Validate(s.bytes.data(), s.bytes.size(), kind, &p, &why), "valid snapshot refused: %s", why.c_str());
    CHECK(p.map.num_levels == (uint32_t) levels && p.map.frame_count == frames, "map header round trip");
    for (int i = 0; i < levels; ++i) {
        CHECK(p.level_payload[i] == s.level_payload[i], "payload offset of level %d", i);
        CHECK(p.map.levels[i].records == s.meta.levels[i].records && p.map.levels[i].num_points == s.meta.levels[i].num_points &&
                  p.map.levels[i].num_touched == s.meta.levels[i].num_touched && p.map.levels[i].cap == s.meta.levels[i].cap,
              "level header round trip %d", i);
    }
    // writing the parsed metadata again gives the same bytes
    {
        std::vector<uint8_t> again(snap::MapHeaderBytes(p.map));
        snap::Writer w(again.data());
        snap::WriteMapHeader(w, p.map);
        CHECK(memcmp(again.data(), s.bytes.data() + s.layout.offset[snap::kSecMap], again.size()) == 0, "map header rewrite");
    }
    CHECK(!Accepts(s.bytes, kind == snap::kKindMap ? snap::kKindOdometry : snap::kKindMap), "kind confusion accepted");
    // truncation: every length below the total (the synthetic snapshots are small), and one byte more
    for (size_t n = 0; n < s.bytes.size(); ++n) CHECK(!Accepts(s.bytes, kind, n), "truncation to %zu accepted", n);
    {
        std::vector<uint8_t> longer = s.bytes;
        longer.push_back(0);
        CHECK(!Accepts(longer, kind), "trailing byte accepted");
    }
    // every section boundary, ±24 bytes, also when the header's total is rewritten to the truncated length
    for (int sec = 0; sec <= snap::kNumSections; ++sec) {
        const uint64_t b = sec < snap::kNumSections ? s.layout.offset[sec] : s.layout.total;
        for (int64_t d = -24; d <= 24; ++d) {
            const int64_t n = (int64_t) b + d;
            if (n < 0 || (uint64_t) n >= s.layout.total) continue;
            std::vector<uint8_t> t(s.bytes.begin(), s.bytes.begin() + n);
            if (n >= (int64_t) snap::kHeaderBytes) {
                const uint64_t total = (uint64_t) n;
                memcpy(t.data() + snap::kChecksumOffset - 8, &total, 8);
                const uint64_t c = snap::Checksum(t.data() + snap::kHeaderBytes, total - snap::kHeaderBytes);
                memcpy(t.data() + snap::kChecksumOffset, &c, 8);
            }
            CHECK(!Accepts(t, kind), "re-checksummed truncation to %lld (section %d) accepted", (long long) n, sec);
        }
    }
    // random single-bit flips anywhere
    std::mt19937_64 rng(seed * 7 + 1);
    for (int k = 0; k < 4000; ++k) {
        std::vector<uint8_t> f = s.bytes;
        const size_t bit = rng() % (8 * f.size());
        f[bit / 8] ^= (uint8_t) (1u << (bit % 8));
        CHECK(!Accepts(f, kind), "bit flip at %zu accepted", bit);
    }
    // magic, version
    {
        Synthetic t = s;
        t.bytes[0] ^= 1;
        CHECK(!Accepts(t.bytes, kind), "wrong magic accepted");
        t = s;
        Put32(t, 8, snap::kVersion + 1);
        CHECK(!Accepts(t.bytes, kind), "wrong version accepted");
    }
    // structural faults with a valid checksum
    const int lv = levels - 1;
    const snap::LevelMeta &L = s.meta.levels[lv];
    CHECK(L.records >= 3, "synthetic level too small");
    {   // slot index >= capacity
        Synthetic t = s;
        Put32(t, RecordAt(t, lv, L.records - 1), (uint32_t) L.cap);
        Reseal(t);
        CHECK(!Accepts(t.bytes, kind), "slot index == capacity accepted");
        Put32(t, RecordAt(t, lv, L.records - 1), 0xFFFFFFFFu);
        Reseal(t);
        CHECK(!Accepts(t.bytes, kind), "slot index 2^32-1 accepted");
    }
    {   // repeated index, decreasing index
        Synthetic t = s;
        Put32(t, RecordAt(t, lv, 1), Get32(t, RecordAt(t, lv, 0)));
        Reseal(t);
        CHECK(!Accepts(t.bytes, kind), "repeated slot index accepted");
        t = s;
        const uint32_t a = Get32(t, RecordAt(t, lv, 1)), b = Get32(t, RecordAt(t, lv, 2));
        Put32(t, RecordAt(t, lv, 1), b);
        Put32(t, RecordAt(t, lv, 2), a);
        Reseal(t);
        CHECK(!Accepts(t.bytes, kind), "decreasing slot index accepted");
    }
    {   // count > B
        Synthetic t = s;
        uint64_t k = 0;
        while (Get32(t, RecordAt(t, lv, k) + 4) == 0) ++k;
        Put32(t, RecordAt(t, lv, k) + 4, L.B + 1);
        Reseal(t);
        CHECK(!Accepts(t.bytes, kind), "count > B accepted");
    }
    {   // totals that disagree with the counters: num_points, num_voxels / num_tombs of the level header
        const size_t hdr = s.layout.offset[snap::kSecMap] + snap::kMapFixedBytes + (size_t) lv * snap::kLevelHeaderBytes;
        Synthetic t = s;
        uint64_t np = L.num_points - 1;
        memcpy(t.bytes.data() + hdr + 16, &np, 8);
        Reseal(t);
        CHECK(!Accepts(t.bytes, kind), "num_points - 1 accepted");
        t = s;
        Put32(t, hdr + 24, L.num_voxels - 1);
        Put32(t, hdr + 28, L.num_tombs + 1);
        Reseal(t);
        CHECK(!Accepts(t.bytes, kind), "voxel / tombstone split moved accepted");
        t = s;   // a tombstone turned into a live voxel without points
        uint64_t k = 0;
        while (Get32(t, RecordAt(t, lv, k) + 4) != 0) ++k;
        uint64_t key = 12345;
        memcpy(t.bytes.data() + RecordAt(t, lv, k) + 8, &key, 8);
        Reseal(t);
        CHECK(!Accepts(t.bytes, kind), "live voxel with zero points accepted");
        t = s;   // capacity not a power of two
        uint64_t cap = L.cap + 1;
        memcpy(t.bytes.data() + hdr, &cap, 8);
        Reseal(t);
        CHECK(!Accepts(t.bytes, kind), "capacity not a power of two accepted");
    }
    {   // a non-finite offset, a frame ordinal beyond the map's frames
        const size_t pts = s.level_payload[lv] + L.records * snap::kRecordBytes;
        Synthetic t = s;
        const float nan = std::numeric_limits<float>::quiet_NaN();
        memcpy(t.bytes.data() + pts + 4, &nan, 4);
        Reseal(t);
        CHECK(!Accepts(t.bytes, kind), "NaN offset accepted");
        t = s;
        const float w = (float) (frames + 1);
        memcpy(t.bytes.data() + pts + 12, &w, 4);
        Reseal(t);
        CHECK(!Accepts(t.bytes, kind), "frame ordinal beyond the map's frames accepted");
    }
    if (kind == snap::kKindOdometry) {   // host state against the trajectory
        Synthetic t = s;
        Put32(t, t.layout.offset[snap::kSecHost], Get32(t, t.layout.offset[snap::kSecHost]) + 1);
        Reseal(t);
        CHECK(!Accepts(t.bytes, kind), "registered frames != trajectory length accepted");
        t = s;
        Put32(t, t.layout.offset[snap::kSecHost] + 8, 0x7fffffff);
        Reseal(t);
        CHECK(!Accepts(t.bytes, kind), "next robust level out of range accepted");
    }
}

// every HostState field written and read back (distinct values, so a swapped or dropped field shows)
static void TestHostStateRoundTrip() {
    snap::HostState a;
    a.registered_frames = 1234;
    a.robust_num_consecutive_failures = 7;
    a.next_robust_level = 3;
    a.suspect_registration_error = 1;
    a.cum_distance = 12.625;
    a.cum_orientation = -3.0625;
    a.skipped_frames = 5;
    a.total_insertions = 999;
    a.last_num_keypoints = 0x123456789ull;
    a.prev_frame_points = 54321;
    a.default_model_present = 1;
    a.default_model_options.model = 2;
    a.default_model_options.log_if_invalid = 1;
    a.default_model_options.beta_location_consistency = 0.5;
    a.default_model_options.beta_constant_velocity = 0.25;
    a.default_model_options.beta_small_velocity = 0.125;
    a.default_model_options.beta_orientation_consistency = 0.0625;
    a.default_model_options.threshold_orientation_deg = 4.5;
    a.default_model_options.threshold_translation_diff = 0.75;
    cticp_frame &f = a.default_model_previous_frame;
    double v = 1.0;
    for (cticp_pose *p : {&f.begin_pose, &f.end_pose}) {
        for (double &q : p->quat) q = (v += 1.0);
        for (double &t : p->tr) t = (v += 1.0);
        p->ref_timestamp = (v += 1.0);
        p->dest_timestamp = (v += 1.0);
        p->ref_frame_id = (uint32_t) (v += 1.0);
        p->dest_frame_id = (uint32_t) (v += 1.0);
    }
    std::vector<uint8_t> buf(snap::kHostStateBytes + 8, 0xCD);
    snap::Writer w(buf.data());
    snap::WriteHostState(w, a);
    CHECK(w.off == snap::kHostStateBytes, "host state wrote %zu of %zu bytes", w.off, snap::kHostStateBytes);
    snap::Reader r(buf.data());
    const snap::HostState b = snap::ReadHostState(r);
    CHECK(r.off == snap::kHostStateBytes, "host state read %zu of %zu bytes", r.off, snap::kHostStateBytes);
    CHECK(b.registered_frames == a.registered_frames, "registered_frames");
    CHECK(b.robust_num_consecutive_failures == a.robust_num_consecutive_failures, "robust_num_consecutive_failures");
    CHECK(b.next_robust_level == a.next_robust_level, "next_robust_level");
    CHECK(b.suspect_registration_error == a.suspect_registration_error, "suspect_registration_error");
    CHECK(b.cum_distance == a.cum_distance && b.cum_orientation == a.cum_orientation, "tracker cumulated motion");
    CHECK(b.skipped_frames == a.skipped_frames && b.total_insertions == a.total_insertions, "tracker counters");
    CHECK(b.last_num_keypoints == a.last_num_keypoints, "last_num_keypoints");
    CHECK(b.prev_frame_points == a.prev_frame_points, "prev_frame_points");
    CHECK(b.default_model_present == a.default_model_present, "default_model_present");
    CHECK(memcmp(&b.default_model_options, &a.default_model_options, sizeof(a.default_model_options)) == 0, "motion model options");
    CHECK(memcmp(&b.default_model_previous_frame, &a.default_model_previous_frame, sizeof(cticp_frame)) == 0, "previous frame");
}

int main() {
    TestHostStateRoundTrip();
    unsigned seed = 1;
    for (int levels = 1; levels <= 3; ++levels)
        for (int normals = 0; normals < 2; ++normals) {
            TestKind(snap::kKindMap, levels, normals != 0, seed++);
            TestKind(snap::kKindOdometry, levels, normals != 0, seed++);
        }
    // the checksum changes under any single-word change (h -> (h ^ w) * P is a bijection per word)
    std::vector<uint8_t> z(4096, 0);
    const uint64_t c0 = snap::Checksum(z.data(), z.size());
    for (size_t i = 0; i < z.size(); i += 97) {
        z[i] = 0x80;
        CHECK(snap::Checksum(z.data(), z.size()) != c0, "checksum blind to byte %zu", i);
        z[i] = 0;
    }
    if (g_failures) {
        printf("SNAPSHOT FORMAT FAILED (%d)\n", g_failures);
        return 1;
    }
    printf("SNAPSHOT FORMAT OK\n");
    return 0;
}
