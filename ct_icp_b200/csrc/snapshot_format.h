// snapshot_format.h — the byte format of odometry and map snapshots (cticp_odometry_save / cticp_map_save), host only.
//
// Plain C++17 (builds with g++ alone, tests/cpp/snapshot_format_test.cpp): layout, writer helpers and the validation that
// runs before a snapshot touches the device. Every field has a fixed width and is little-endian; nothing is written as a raw
// C++ struct except the ABI option structs of include/cticp.h, whose layout the ABI already fixes.
//
//   header (kHeaderBytes)
//     u64 magic | u32 version | u32 kind | u64 section size × kNumSections | u64 total size | u64 checksum of the payload
//   payload, the sections in order:
//     options     cticp_odometry_options bytes (odometry snapshots; empty for a map)
//     host state  the engine state a later frame reads (kHostStateBytes; empty for a map)
//     trajectory  u64 count, then count cticp_frames field by field (empty for a map)
//     map         cticp_map_options bytes | u32 levels | u32 has_normals | u64 frame_count | per level a kLevelHeaderBytes
//                 header, then per level its payload: records (u32 slot, u32 count, u64 key) in slot order, the live
//                 voxels' points (float4: offsets from the voxel origin, w = ±(source frame ordinal + 1)) contiguous in the
//                 same order, and, when the map keeps normals, one voxel normal (4 × f64) per record
//     origins     3 × f64 per inserted frame (frame_count of them) when the map keeps normals, else empty
// A record is every non-empty slot of the table: live voxels and tombstones (count 0), so a load puts every slot back at its
// own index and load → save reproduces the bytes.
#pragma once
#include <cmath>
#include <cstddef>
#include <cstdint>
#include <cstring>
#include <string>
#include <vector>

#include "../../include/cticp.h"

#if defined(__BYTE_ORDER__) && __BYTE_ORDER__ != __ORDER_LITTLE_ENDIAN__
#error "the snapshot format is little-endian; big-endian hosts are not supported"
#endif

namespace cticp {
namespace snap {

constexpr uint64_t kMagic = 0x50414E5350434954ull;   // "TICPSNAP" read as little-endian bytes
constexpr uint32_t kVersion = 1;
constexpr uint32_t kKindOdometry = 1, kKindMap = 2;
enum { kSecOptions = 0, kSecHost, kSecTrajectory, kSecMap, kSecOrigins, kNumSections };
constexpr size_t kHeaderBytes = 8 + 4 + 4 + 8 * kNumSections + 8 + 8;
constexpr size_t kChecksumOffset = kHeaderBytes - 8;
constexpr size_t kFrameBytes = 2 * (7 * 8 + 2 * 8 + 2 * 4);   // cticp_frame, field by field
constexpr size_t kRecordBytes = 16, kPointBytes = 16, kNormalBytes = 32;
constexpr size_t kLevelHeaderBytes = 48;
constexpr size_t kMapFixedBytes = sizeof(cticp_map_options) + 4 + 4 + 8;
constexpr uint64_t kKeyEmpty = ~0ull, kKeyTomb = ~0ull - 1ull;   // device_map.cuh kEmptyKey / kTombKey
constexpr int kMaxB = 64;                                         // max_num_points a map level supports
constexpr uint64_t kMaxCap = 1ull << 31;
constexpr int32_t kMaxRobustLevel = 1 << 16;   // a robust level a snapshot may carry (each level is one more attempt)

// 64-bit checksum of a byte range, word by word: h = (h ^ w) · P over little-endian 64-bit words (the tail zero-padded),
// then the length. Each step is a bijection of h for a fixed word, so any change confined to one word changes the result.
inline uint64_t Checksum(const uint8_t *p, size_t n) {
    uint64_t h = 0xcbf29ce484222325ull;
    const uint64_t P = 0x100000001b3ull * 0x9E3779B97F4A7C15ull | 1ull;
    size_t i = 0;
    for (; i + 8 <= n; i += 8) {
        uint64_t w;
        memcpy(&w, p + i, 8);
        h = (h ^ w) * P;
    }
    if (i < n) {
        uint64_t w = 0;
        memcpy(&w, p + i, n - i);
        h = (h ^ w) * P;
    }
    h = (h ^ (uint64_t) n) * P;
    return h ^ (h >> 29);
}

// ---- fixed-width little-endian fields ---------------------------------------------------------------------------------
struct Writer {
    uint8_t *p;
    size_t off = 0;
    explicit Writer(uint8_t *dst, size_t at = 0) : p(dst), off(at) {}
    void bytes(const void *src, size_t n) { memcpy(p + off, src, n); off += n; }
    void u32(uint32_t v) { bytes(&v, 4); }
    void i32(int32_t v) { bytes(&v, 4); }
    void u64(uint64_t v) { bytes(&v, 8); }
    void f64(double v) { bytes(&v, 8); }
    void pose(const cticp_pose &c) {
        for (int i = 0; i < 4; ++i) f64(c.quat[i]);
        for (int i = 0; i < 3; ++i) f64(c.tr[i]);
        f64(c.ref_timestamp); f64(c.dest_timestamp);
        u32(c.ref_frame_id); u32(c.dest_frame_id);
    }
    void frame(const cticp_frame &f) { pose(f.begin_pose); pose(f.end_pose); }
};
struct Reader {
    const uint8_t *p;
    size_t off = 0;
    explicit Reader(const uint8_t *src, size_t at = 0) : p(src), off(at) {}
    void bytes(void *dst, size_t n) { memcpy(dst, p + off, n); off += n; }
    uint32_t u32() { uint32_t v; bytes(&v, 4); return v; }
    int32_t i32() { int32_t v; bytes(&v, 4); return v; }
    uint64_t u64() { uint64_t v; bytes(&v, 8); return v; }
    double f64() { double v; bytes(&v, 8); return v; }
    cticp_pose pose() {
        cticp_pose c;
        for (int i = 0; i < 4; ++i) c.quat[i] = f64();
        for (int i = 0; i < 3; ++i) c.tr[i] = f64();
        c.ref_timestamp = f64(); c.dest_timestamp = f64();
        c.ref_frame_id = u32(); c.dest_frame_id = u32();
        return c;
    }
    cticp_frame frame() {
        cticp_frame f;
        f.begin_pose = pose();
        f.end_pose = pose();
        return f;
    }
};

// ---- host state: every member of the engine a later frame reads ---------------------------------------------------------
struct HostState {
    int32_t registered_frames = 0;
    int32_t robust_num_consecutive_failures = 0;
    int32_t next_robust_level = 0;
    int32_t suspect_registration_error = 0;
    double cum_distance = 0, cum_orientation = 0;   // tracker_
    int32_t skipped_frames = 0, total_insertions = 0;
    uint64_t last_num_keypoints = 0;                 // grid-size hint of the ICP kernels (Engine::KeypointHint)
    int32_t prev_frame_points = 0;                   // the previous frame's sub-sampled point count (Engine::ArmTail)
    int32_t default_model_present = 0;               // default_motion_model_
    cticp_motion_model_options default_model_options{};
    cticp_frame default_model_previous_frame{};
};
constexpr size_t kHostStateBytes = 4 * 4 + 2 * 8 + 2 * 4 + 8 + 4 + 4 + sizeof(cticp_motion_model_options) + kFrameBytes;

inline void WriteHostState(Writer &w, const HostState &s) {
    w.i32(s.registered_frames); w.i32(s.robust_num_consecutive_failures); w.i32(s.next_robust_level);
    w.i32(s.suspect_registration_error);
    w.f64(s.cum_distance); w.f64(s.cum_orientation);
    w.i32(s.skipped_frames); w.i32(s.total_insertions);
    w.u64(s.last_num_keypoints);
    w.i32(s.default_model_present); w.i32(s.prev_frame_points);
    w.bytes(&s.default_model_options, sizeof(s.default_model_options));
    w.frame(s.default_model_previous_frame);
}
inline HostState ReadHostState(Reader &r) {
    HostState s;
    s.registered_frames = r.i32(); s.robust_num_consecutive_failures = r.i32(); s.next_robust_level = r.i32();
    s.suspect_registration_error = r.i32();
    s.cum_distance = r.f64(); s.cum_orientation = r.f64();
    s.skipped_frames = r.i32(); s.total_insertions = r.i32();
    s.last_num_keypoints = r.u64();
    s.default_model_present = r.i32(); s.prev_frame_points = r.i32();
    r.bytes(&s.default_model_options, sizeof(s.default_model_options));
    s.default_model_previous_frame = r.frame();
    return s;
}

// ---- the map section --------------------------------------------------------------------------------------------------
struct LevelMeta {
    uint64_t cap = 0;          // slots (a power of two)
    uint32_t B = 0;            // max_num_points
    uint64_t num_points = 0;   // MapCounters
    uint32_t num_voxels = 0, num_tombs = 0, num_touched = 0, overflow = 0;
    uint64_t records = 0;      // non-empty slots: num_voxels + num_tombs
};
struct MapMeta {
    cticp_map_options options{};
    uint32_t num_levels = 0;
    uint32_t has_normals = 0;
    uint64_t frame_count = 0;
    LevelMeta levels[CTICP_MAX_RESOLUTIONS];
};
// bytes of one level's payload
inline uint64_t LevelPayloadBytes(const LevelMeta &L, bool normals) {
    return L.records * (kRecordBytes + (normals ? kNormalBytes : 0)) + L.num_points * kPointBytes;
}
inline uint64_t MapHeaderBytes(const MapMeta &m) { return kMapFixedBytes + (uint64_t) m.num_levels * kLevelHeaderBytes; }
inline uint64_t MapSectionBytes(const MapMeta &m) {
    uint64_t n = MapHeaderBytes(m);
    for (uint32_t i = 0; i < m.num_levels; ++i) n += LevelPayloadBytes(m.levels[i], m.has_normals != 0);
    return n;
}
inline uint64_t OriginsBytes(const MapMeta &m) { return m.has_normals ? 24 * m.frame_count : 0; }

inline void WriteMapHeader(Writer &w, const MapMeta &m) {
    w.bytes(&m.options, sizeof(m.options));
    w.u32(m.num_levels); w.u32(m.has_normals); w.u64(m.frame_count);
    for (uint32_t i = 0; i < m.num_levels; ++i) {
        const LevelMeta &L = m.levels[i];
        w.u64(L.cap); w.u32(L.B); w.u32(0);
        w.u64(L.num_points); w.u32(L.num_voxels); w.u32(L.num_tombs); w.u32(L.num_touched); w.u32(L.overflow);
        w.u64(L.records);
    }
}

// ---- the whole snapshot ------------------------------------------------------------------------------------------------
struct Layout {
    uint32_t kind = 0;
    uint64_t size[kNumSections] = {};
    uint64_t offset[kNumSections] = {};   // from the start of the snapshot
    uint64_t total = 0;
};
inline Layout MakeLayout(uint32_t kind, const uint64_t (&size)[kNumSections]) {
    Layout l;
    l.kind = kind;
    uint64_t at = kHeaderBytes;
    for (int s = 0; s < kNumSections; ++s) {
        l.size[s] = size[s];
        l.offset[s] = at;
        at += size[s];
    }
    l.total = at;
    return l;
}
inline void WriteHeader(uint8_t *dst, const Layout &l) {
    Writer w(dst);
    w.u64(kMagic); w.u32(kVersion); w.u32(l.kind);
    for (int s = 0; s < kNumSections; ++s) w.u64(l.size[s]);
    w.u64(l.total);
    w.u64(0);   // checksum: Seal
}
// after every section is written
inline void Seal(uint8_t *dst, const Layout &l) {
    const uint64_t c = Checksum(dst + kHeaderBytes, l.total - kHeaderBytes);
    memcpy(dst + kChecksumOffset, &c, 8);
}

// What a validated snapshot holds; pointers into the caller's bytes.
struct Parsed {
    Layout layout;
    MapMeta map;
    const uint8_t *base = nullptr;
    uint64_t level_payload[CTICP_MAX_RESOLUTIONS] = {};   // offset of each level's payload from base
    uint64_t map_payload = 0, map_payload_bytes = 0;       // all levels' payloads, contiguous
};

inline bool Fail(std::string *why, const char *msg) {
    if (why) *why = msg;
    return false;
}

// Whether an odometry with these options keeps per-voxel normals: only the distance-based strategy's sensor-side filter
// reads them (Engine::Engine)
inline bool NeedsNormals(const cticp_odometry_options &o) {
    return o.map_options.select_valid_normals_direction && o.neighborhood_strategy.type == CTICP_STRATEGY_DISTANCE_BASED;
}
// map options equal field by field (the explicit padding fields excluded)
inline bool SameMapOptions(const cticp_map_options &a, const cticp_map_options &b) {
    if (a.num_resolutions != b.num_resolutions || a.select_valid_normals_direction != b.select_valid_normals_direction ||
        a.max_frames_to_keep != b.max_frames_to_keep || a.default_radius != b.default_radius ||
        a.capacity_voxels != b.capacity_voxels)
        return false;
    for (int i = 0; i < CTICP_MAX_RESOLUTIONS; ++i) {
        const cticp_resolution_param &x = a.resolutions[i], &y = b.resolutions[i];
        if (x.resolution != y.resolution || x.min_distance_between_points != y.min_distance_between_points ||
            x.max_num_points != y.max_num_points)
            return false;
    }
    return true;
}

// The map section at [off, off + n) of base: header fields, then the structure of every level's payload. Nothing may be
// taken from the payload until this has passed.
inline bool ValidateMap(const uint8_t *base, uint64_t off, uint64_t n, Parsed *out, std::string *why) {
    if (n < kMapFixedBytes) return Fail(why, "snapshot: map section too short");
    Reader r(base, off);
    MapMeta &m = out->map;
    r.bytes(&m.options, sizeof(m.options));
    m.num_levels = r.u32(); m.has_normals = r.u32(); m.frame_count = r.u64();
    if (m.num_levels < 1 || m.num_levels > CTICP_MAX_RESOLUTIONS || (int) m.num_levels != m.options.num_resolutions)
        return Fail(why, "snapshot: map level count out of range or not the map options'");
    if (m.has_normals > 1) return Fail(why, "snapshot: bad normals flag");
    if (m.frame_count >= (1u << 24)) return Fail(why, "snapshot: frame count out of range");
    if (n < MapHeaderBytes(m)) return Fail(why, "snapshot: map section too short for its level headers");
    for (uint32_t i = 0; i < m.num_levels; ++i) {
        LevelMeta &L = m.levels[i];
        L.cap = r.u64(); L.B = r.u32(); const uint32_t pad = r.u32();
        L.num_points = r.u64(); L.num_voxels = r.u32(); L.num_tombs = r.u32(); L.num_touched = r.u32(); L.overflow = r.u32();
        L.records = r.u64();
        const auto &rp = m.options.resolutions[i];
        if (pad != 0 || L.cap < 1024 || L.cap > kMaxCap || (L.cap & (L.cap - 1)) != 0)
            return Fail(why, "snapshot: table capacity is not a power of two in range");
        if ((int) L.B != rp.max_num_points || L.B < 1 || L.B > (uint32_t) kMaxB)
            return Fail(why, "snapshot: max_num_points disagrees with the map options");
        if (!(rp.resolution > 0) || L.overflow > 1)
            return Fail(why, "snapshot: bad level header");
        if (L.records != (uint64_t) L.num_voxels + L.num_tombs || L.records > L.cap)
            return Fail(why, "snapshot: record count disagrees with the counters");
        if (L.num_points > (uint64_t) L.num_voxels * L.B || L.num_points >= (1ull << 32))
            return Fail(why, "snapshot: more points than the voxels hold");
    }
    if (MapSectionBytes(m) != n) return Fail(why, "snapshot: map section size disagrees with its counters");
    out->map_payload = off + MapHeaderBytes(m);
    out->map_payload_bytes = n - MapHeaderBytes(m);
    // the structure of every level: slots strictly increasing and below the capacity, counts <= B, a tombstone empty and
    // a live voxel not, totals that match the counters, finite offsets and frame ordinals that exist
    uint64_t at = out->map_payload;
    for (uint32_t i = 0; i < m.num_levels; ++i) {
        const LevelMeta &L = m.levels[i];
        out->level_payload[i] = at;
        const uint8_t *rec = base + at, *pts = rec + L.records * kRecordBytes;
        uint64_t points = 0, voxels = 0, tombs = 0;
        int64_t prev = -1;
        for (uint64_t k = 0; k < L.records; ++k) {
            uint32_t slot, count;
            uint64_t key;
            memcpy(&slot, rec + k * kRecordBytes, 4);
            memcpy(&count, rec + k * kRecordBytes + 4, 4);
            memcpy(&key, rec + k * kRecordBytes + 8, 8);
            if ((int64_t) slot <= prev || slot >= L.cap) return Fail(why, "snapshot: slot index out of order or out of range");
            prev = slot;
            if (count > L.B) return Fail(why, "snapshot: voxel holds more points than max_num_points");
            if (key == kKeyEmpty) return Fail(why, "snapshot: record of an empty slot");
            if (key == kKeyTomb) {
                if (count != 0) return Fail(why, "snapshot: tombstone with points");
                ++tombs;
                continue;
            }
            if (count == 0) return Fail(why, "snapshot: live voxel without points");
            if (points + count > L.num_points) return Fail(why, "snapshot: point total disagrees with the counters");
            for (uint32_t j = 0; j < count; ++j) {
                float q[4];
                memcpy(q, pts + (points + j) * kPointBytes, 16);
                if (!(std::isfinite(q[0]) && std::isfinite(q[1]) && std::isfinite(q[2])))
                    return Fail(why, "snapshot: non-finite point offset");
                const float a = std::fabs(q[3]);
                if (!(a >= 1.f && a <= (float) (1u << 24)) || a != std::floor(a) || (uint64_t) a > m.frame_count)
                    return Fail(why, "snapshot: point with a frame ordinal the map never inserted");
            }
            points += count;
            ++voxels;
        }
        if (points != L.num_points || voxels != L.num_voxels || tombs != L.num_tombs)
            return Fail(why, "snapshot: totals disagree with the counters");
        at += LevelPayloadBytes(L, m.has_normals != 0);
    }
    return true;
}

// Header, sizes and checksum, then the structure of every section. `expect_kind`: kKindOdometry or kKindMap.
inline bool Validate(const void *src, size_t n_bytes, uint32_t expect_kind, Parsed *out, std::string *why) {
    const uint8_t *p = static_cast<const uint8_t *>(src);
    if (!p || n_bytes < kHeaderBytes) return Fail(why, "snapshot: shorter than its header");
    Reader r(p);
    if (r.u64() != kMagic) return Fail(why, "snapshot: bad magic");
    if (r.u32() != kVersion) return Fail(why, "snapshot: unsupported format version");
    const uint32_t kind = r.u32();
    if (kind != expect_kind) return Fail(why, "snapshot: an odometry snapshot and a map snapshot are not interchangeable");
    uint64_t size[kNumSections];
    uint64_t sum = kHeaderBytes;
    for (int s = 0; s < kNumSections; ++s) {
        size[s] = r.u64();
        if (size[s] > n_bytes) return Fail(why, "snapshot: section larger than the snapshot");
        sum += size[s];
    }
    const uint64_t total = r.u64();
    uint64_t checksum = r.u64();
    if (total != n_bytes || sum != total) return Fail(why, "snapshot: size disagrees with its header (truncated?)");
    if (Checksum(p + kHeaderBytes, total - kHeaderBytes) != checksum) return Fail(why, "snapshot: checksum mismatch");
    out->layout = MakeLayout(kind, size);
    out->base = p;
    const Layout &l = out->layout;
    if (kind == kKindOdometry) {
        if (l.size[kSecOptions] != sizeof(cticp_odometry_options)) return Fail(why, "snapshot: options section size");
        if (l.size[kSecHost] != kHostStateBytes) return Fail(why, "snapshot: host state section size");
        if (l.size[kSecTrajectory] < 8) return Fail(why, "snapshot: trajectory section size");
        Reader t(p, l.offset[kSecTrajectory]);
        const uint64_t frames = t.u64();
        if (frames > (l.size[kSecTrajectory] - 8) / kFrameBytes || 8 + frames * kFrameBytes != l.size[kSecTrajectory])
            return Fail(why, "snapshot: trajectory section size");
    } else if (l.size[kSecOptions] || l.size[kSecHost] || l.size[kSecTrajectory]) {
        return Fail(why, "snapshot: a map snapshot has only the map and origins sections");
    }
    if (!ValidateMap(p, l.offset[kSecMap], l.size[kSecMap], out, why)) return false;
    if (l.size[kSecOrigins] != OriginsBytes(out->map)) return Fail(why, "snapshot: origins section size");
    for (uint64_t i = 0; i < 3 * (l.size[kSecOrigins] / 24); ++i) {
        double v;
        memcpy(&v, p + l.offset[kSecOrigins] + 8 * i, 8);
        if (!std::isfinite(v)) return Fail(why, "snapshot: non-finite frame origin");
    }
    if (kind == kKindOdometry) {
        cticp_odometry_options o;
        memcpy(&o, p + l.offset[kSecOptions], sizeof(o));
        if (!SameMapOptions(o.map_options, out->map.options))
            return Fail(why, "snapshot: map section options disagree with the odometry options");
        Reader h(p, l.offset[kSecHost]);
        const HostState s = ReadHostState(h);
        Reader t(p, l.offset[kSecTrajectory]);
        if (s.registered_frames < 0 || (uint64_t) s.registered_frames != t.u64())
            return Fail(why, "snapshot: registered frame count disagrees with the trajectory");
        if (s.robust_num_consecutive_failures < 0 || s.next_robust_level < 0 || s.next_robust_level > kMaxRobustLevel ||
            s.suspect_registration_error > 1 || s.suspect_registration_error < 0 || s.skipped_frames < 0 ||
            s.total_insertions < 0 || s.prev_frame_points < 0 || s.default_model_present < 0 || s.default_model_present > 1 ||
            s.last_num_keypoints > (1ull << 32) || !std::isfinite(s.cum_distance) || !std::isfinite(s.cum_orientation))
            return Fail(why, "snapshot: host state out of range");
        if (out->map.has_normals != (NeedsNormals(o) ? 1u : 0u))
            return Fail(why, "snapshot: normals flag disagrees with the odometry options");
    }
    return true;
}

}  // namespace snap
}  // namespace cticp
