// snapshot.cu — save, load and clone of voxel maps and odometry handles (snapshot_format.h has the byte format).
//
// Device side: k_snapshot_pack compacts a level's non-empty slots, their point runs and their normals into a contiguous
// buffer in slot order; k_snapshot_unpack scatters them back, every slot to its own index and every run to slot · B. Both
// take the offsets from a prefix over tiles of 1024 slots (records) with the sampler's decoupled look-back
// (tile_lookback.cuh), tiles handed out in launch order from an atomic ticket.
#include "engine.h"
#include "snapshot_format.h"
#include "tile_lookback.cuh"

#include <algorithm>
#include <cstring>

namespace cticp {

constexpr int kSnapThreads = 256, kSnapPer = 4, kSnapTile = kSnapThreads * kSnapPer, kSnapWarps = kSnapThreads / 32;
// the unpack's tiles are records, not slots: a map holds far fewer records than slots (load <= 0.5), so one record per
// thread spreads its scatter over four times as many CTAs
constexpr int kUnpackPer = 1, kUnpackTile = kSnapThreads * kUnpackPer;

struct SnapScratch {
    uint32_t warp_rec[kSnapWarps], warp_pts[kSnapWarps];
    uint32_t before_rec, before_pts, tile_rec;
    int tile;
    // per record of the tile (by its rank in the tile): its point count, where its run starts in the table (slot, times B)
    // and in the payload
    uint32_t count[kSnapTile];
    uint32_t slot[kSnapTile];
    uint32_t run[kSnapTile];
};

// Inclusive warp scans of two counters, the CTA's exclusive offsets of this thread, the tile's look-back. Returns this
// thread's exclusive (records, points) offsets within the whole level; `last`: the tile that writes the totals.
__device__ __forceinline__ void snap_tile_prefix(uint32_t r, uint32_t p, int tile, bool last, unsigned long long *desc_rec,
                                                 unsigned long long *desc_pts, unsigned *totals, SnapScratch &sc,
                                                 uint32_t *rec_off, uint32_t *pts_off) {
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    uint32_t ir = r, ip = p;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const uint32_t yr = __shfl_up_sync(0xffffffffu, ir, o), yp = __shfl_up_sync(0xffffffffu, ip, o);
        if (lane >= o) { ir += yr; ip += yp; }
    }
    if (lane == 31) { sc.warp_rec[w] = ir; sc.warp_pts[w] = ip; }
    __syncthreads();
    if (w == 0) {
        const uint32_t wr = lane < kSnapWarps ? sc.warp_rec[lane] : 0u, wp = lane < kSnapWarps ? sc.warp_pts[lane] : 0u;
        uint32_t er = wr, ep = wp;   // inclusive over the warps, then exclusive
#pragma unroll
        for (int o = 1; o < kSnapWarps; o <<= 1) {
            const uint32_t yr = __shfl_up_sync(0xffffffffu, er, o), yp = __shfl_up_sync(0xffffffffu, ep, o);
            if (lane >= o) { er += yr; ep += yp; }
        }
        const uint32_t tile_r = __shfl_sync(0xffffffffu, er, kSnapWarps - 1), tile_p = __shfl_sync(0xffffffffu, ep, kSnapWarps - 1);
        const uint32_t before_r = desc_rec ? tile_lookback(desc_rec, tile, tile_r) : 0u;
        const uint32_t before_p = tile_lookback(desc_pts, tile, tile_p);
        __syncwarp();
        if (lane < kSnapWarps) { sc.warp_rec[lane] = er - wr; sc.warp_pts[lane] = ep - wp; }
        if (lane == 0) {
            sc.before_rec = before_r;
            sc.before_pts = before_p;
            sc.tile_rec = tile_r;
            if (last) { totals[0] = before_r + tile_r; totals[1] = before_p + tile_p; }
        }
    }
    __syncthreads();
    *rec_off = sc.before_rec + sc.warp_rec[w] + (ir - r);
    *pts_off = sc.before_pts + sc.warp_pts[w] + (ip - p);
}

// The runs of the tile's records, one warp per record, lanes over its points (<= 64 float4: two coalesced rounds)
template <bool kToPayload>
__device__ __forceinline__ void snap_copy_runs(float4 *__restrict__ table, int B, float4 *__restrict__ payload, uint32_t n_rec,
                                               const SnapScratch &sc) {
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    for (uint32_t k = w; k < n_rec; k += kSnapWarps) {
        const uint32_t c = sc.count[k];
        const size_t t = (size_t) sc.slot[k] * B, p = sc.run[k];
        for (uint32_t j = lane; j < c; j += 32) {
            if (kToPayload) payload[p + j] = table[t + j];
            else table[t + j] = payload[p + j];
        }
    }
}

// Pack one level: records (slot, count, key) | points | normals (one per record), each contiguous in slot order.
__global__ void __launch_bounds__(kSnapThreads)
k_snapshot_pack(MapLevel L, unsigned long long *desc_rec, unsigned long long *desc_pts, unsigned *ticket, unsigned *totals,
                uint4 *__restrict__ out_rec, float4 *__restrict__ out_pts, double2 *__restrict__ out_nrm) {
    __shared__ SnapScratch sc;
    const uint32_t cap = L.cap_mask + 1;
    const int num_tiles = (int) ((cap + kSnapTile - 1) / kSnapTile);
    for (;;) {
        __syncthreads();   // scratch reuse across tiles
        if (threadIdx.x == 0) sc.tile = (int) atomicAdd(ticket, 1u);
        __syncthreads();
        const int tile = sc.tile;
        if (tile >= num_tiles) return;
        const uint32_t s0 = (uint32_t) tile * kSnapTile + threadIdx.x * kSnapPer;
        uint4 raw[kSnapPer];
        uint32_t r = 0, p = 0;
#pragma unroll
        for (int k = 0; k < kSnapPer; ++k) {
            raw[k] = s0 + k < cap ? *reinterpret_cast<const uint4 *>(L.slots + s0 + k) : make_uint4(0xffffffffu, 0xffffffffu, 0u, 0u);
            const unsigned long long key = (unsigned long long) raw[k].x | ((unsigned long long) raw[k].y << 32);
            if (key != kEmptyKey) {
                ++r;
                p += key == kTombKey ? 0u : raw[k].z;
            }
        }
        uint32_t ro, po;
        snap_tile_prefix(r, p, tile, tile == num_tiles - 1, desc_rec, desc_pts, totals, sc, &ro, &po);
#pragma unroll
        for (int k = 0; k < kSnapPer; ++k) {
            const unsigned long long key = (unsigned long long) raw[k].x | ((unsigned long long) raw[k].y << 32);
            if (key == kEmptyKey) continue;
            const uint32_t s = s0 + k, c = key == kTombKey ? 0u : raw[k].z;
            out_rec[ro] = make_uint4(s, c, raw[k].x, raw[k].y);
            if (out_nrm && L.normals) {
                const double2 *n = reinterpret_cast<const double2 *>(L.normals + 4 * (size_t) s);
                out_nrm[2 * (size_t) ro] = n[0];
                out_nrm[2 * (size_t) ro + 1] = n[1];
            }
            const uint32_t li = ro - sc.before_rec;
            sc.count[li] = c;
            sc.slot[li] = s;
            sc.run[li] = po;
            ++ro;
            po += c;
        }
        __syncthreads();
        snap_copy_runs<true>(L.points, L.B, out_pts, sc.tile_rec, sc);
    }
}

// Unpack one level into a cleared table: every record to its slot, its normal next to it, its run to slot · B. The records
// passed snap::ValidateMap (slots distinct and below the capacity, counts <= B, runs that add up to the payload's points).
__global__ void __launch_bounds__(kSnapThreads)
k_snapshot_unpack(MapLevel L, uint32_t n_rec, unsigned long long *desc_pts, unsigned *ticket, unsigned *totals,
                  const uint4 *__restrict__ in_rec, const float4 *__restrict__ in_pts, const double2 *__restrict__ in_nrm) {
    __shared__ SnapScratch sc;
    const int num_tiles = (int) ((n_rec + kUnpackTile - 1) / kUnpackTile);
    for (;;) {
        __syncthreads();
        if (threadIdx.x == 0) sc.tile = (int) atomicAdd(ticket, 1u);
        __syncthreads();
        const int tile = sc.tile;
        if (tile >= num_tiles) return;
        const uint32_t r0 = (uint32_t) tile * kUnpackTile + threadIdx.x * kUnpackPer;
        uint4 rec[kUnpackPer];
        uint32_t r = 0, p = 0;
#pragma unroll
        for (int k = 0; k < kUnpackPer; ++k) {
            rec[k] = r0 + k < n_rec ? in_rec[r0 + k] : make_uint4(0u, 0u, 0u, 0u);
            if (r0 + k < n_rec) {
                ++r;
                p += rec[k].y;
            }
        }
        uint32_t ro, po;
        snap_tile_prefix(r, p, tile, tile == num_tiles - 1, nullptr, desc_pts, totals, sc, &ro, &po);
        const uint32_t base = (uint32_t) tile * kUnpackTile;
#pragma unroll
        for (int k = 0; k < kUnpackPer; ++k) {
            if (r0 + k >= n_rec) continue;
            const uint32_t s = rec[k].x, c = rec[k].y;
            MapSlot v;
            v.key = (unsigned long long) rec[k].z | ((unsigned long long) rec[k].w << 32);
            v.count = c;
            v._pad = 0;
            L.slots[s] = v;
            if (in_nrm && L.normals) {
                double2 *n = reinterpret_cast<double2 *>(L.normals + 4 * (size_t) s);
                n[0] = in_nrm[2 * (size_t) (r0 + k)];
                n[1] = in_nrm[2 * (size_t) (r0 + k) + 1];
            }
            const uint32_t li = r0 + k - base;
            sc.count[li] = c;
            sc.slot[li] = s;
            sc.run[li] = po;
            po += c;
        }
        __syncthreads();
        snap_copy_runs<false>(L.points, L.B, const_cast<float4 *>(in_pts), min((uint32_t) kUnpackTile, n_rec - base), sc);
    }
}

// ---- DeviceMap ----------------------------------------------------------------------------------------------------------
snap::MapMeta DeviceMap::SnapshotMeta() const {
    // the device counters, read without touching the host copy the next frame's table maintenance reads
    MapCounters c[CTICP_MAX_RESOLUTIONS];
    CT_CUDA_CHECK(cudaMemcpyAsync(c, d_counters_.data(), sizeof(MapCounters) * levels_.size(), cudaMemcpyDeviceToHost, stream_));
    CT_CUDA_CHECK(cudaStreamSynchronize(stream_));
    snap::MapMeta m;
    m.options = options_;
    m.num_levels = (uint32_t) levels_.size();
    m.has_normals = with_normals_ ? 1u : 0u;
    m.frame_count = frame_count_;
    for (size_t i = 0; i < levels_.size(); ++i) {
        snap::LevelMeta &L = m.levels[i];
        L.cap = (uint64_t) levels_[i].cap_mask + 1;
        L.B = (uint32_t) levels_[i].B;
        L.num_points = c[i].num_points;
        L.num_voxels = c[i].num_voxels;
        L.num_tombs = c[i].num_tombs;
        L.num_touched = c[i].num_touched;
        L.overflow = c[i].overflow;
        L.records = (uint64_t) c[i].num_voxels + c[i].num_tombs;
        if (L.num_points >= (1ull << 32)) throw CapacityError("snapshot: a map level holds 2^32 points or more");
    }
    return m;
}

// scratch of one pack / unpack: the two descriptor arrays, the ticket, the two totals
struct SnapLaunchScratch {
    DeviceArray<unsigned long long> words;
    size_t tiles = 0;
    void Prepare(size_t items, size_t tile, cudaStream_t stream) {
        tiles = std::max<size_t>(1, (items + tile - 1) / tile);
        words.reserve(2 * tiles + 2, stream);
        CT_CUDA_CHECK(cudaMemsetAsync(words.data(), 0, sizeof(unsigned long long) * (2 * tiles + 2), stream));
    }
    unsigned long long *desc_rec() const { return words.data(); }
    unsigned long long *desc_pts() const { return words.data() + tiles; }
    unsigned *ticket() const { return reinterpret_cast<unsigned *>(words.data() + 2 * tiles); }
    unsigned *totals() const { return reinterpret_cast<unsigned *>(words.data() + 2 * tiles + 1); }
};

static int SnapGrid(size_t tiles) {
    int dev = 0, sms = 132;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    return (int) std::max<size_t>(1, std::min<size_t>(tiles, (size_t) sms * 8));
}

void DeviceMap::Pack(unsigned char *d_out, const snap::MapMeta &meta) {
    SnapLaunchScratch sc;
    size_t at = 0;
    std::vector<unsigned> totals(2 * levels_.size());
    for (size_t i = 0; i < levels_.size(); ++i) {
        const snap::LevelMeta &L = meta.levels[i];
        uint4 *rec = reinterpret_cast<uint4 *>(d_out + at);
        float4 *pts = reinterpret_cast<float4 *>(d_out + at + L.records * snap::kRecordBytes);
        double2 *nrm = with_normals_ ? reinterpret_cast<double2 *>(d_out + at + L.records * snap::kRecordBytes +
                                                                     L.num_points * snap::kPointBytes)
                                     : nullptr;
        at += snap::LevelPayloadBytes(L, with_normals_);
        sc.Prepare(L.cap, kSnapTile, stream_);
        k_snapshot_pack<<<SnapGrid(sc.tiles), kSnapThreads, 0, stream_>>>(levels_[i], sc.desc_rec(), sc.desc_pts(), sc.ticket(),
                                                                          sc.totals(), rec, pts, nrm);
        CT_CUDA_CHECK(cudaGetLastError());
        CT_CUDA_CHECK(cudaMemcpyAsync(totals.data() + 2 * i, sc.totals(), 2 * sizeof(unsigned), cudaMemcpyDeviceToHost, stream_));
        CT_CUDA_CHECK(cudaStreamSynchronize(stream_));   // (the scratch of the next level reuses the words)
    }
    for (size_t i = 0; i < levels_.size(); ++i)
        if (totals[2 * i] != meta.levels[i].records || totals[2 * i + 1] != meta.levels[i].num_points)
            throw std::runtime_error("snapshot: the packed totals of map level " + std::to_string(i) + " disagree with its counters");
}

void DeviceMap::Unpack(const unsigned char *d_payload, const snap::MapMeta &meta, const double *origins) {
    // every level cleared (k_clear_level), at the snapshot's capacity
    Clear();
    for (size_t i = 0; i < levels_.size(); ++i) {
        const uint64_t cap = meta.levels[i].cap;
        if (cap == (uint64_t) levels_[i].cap_mask + 1) continue;
        MapLevel fresh{};
        LevelStorage storage = AllocLevel(fresh, (uint32_t) cap, options_.resolutions[i]);
        CT_CUDA_CHECK(cudaStreamSynchronize(stream_));   // (the old tables may still be cleared)
        levels_[i] = fresh;
        storage_[i] = std::move(storage);
    }
    SnapLaunchScratch sc;
    size_t at = 0;
    std::vector<unsigned> totals(2 * levels_.size());
    for (size_t i = 0; i < levels_.size(); ++i) {
        const snap::LevelMeta &L = meta.levels[i];
        const uint4 *rec = reinterpret_cast<const uint4 *>(d_payload + at);
        const float4 *pts = reinterpret_cast<const float4 *>(d_payload + at + L.records * snap::kRecordBytes);
        const double2 *nrm = meta.has_normals ? reinterpret_cast<const double2 *>(d_payload + at + L.records * snap::kRecordBytes +
                                                                                    L.num_points * snap::kPointBytes)
                                              : nullptr;
        at += snap::LevelPayloadBytes(L, meta.has_normals != 0);
        totals[2 * i] = totals[2 * i + 1] = 0;
        if (L.records == 0) continue;
        sc.Prepare(L.records, kUnpackTile, stream_);
        k_snapshot_unpack<<<SnapGrid(sc.tiles), kSnapThreads, 0, stream_>>>(levels_[i], (uint32_t) L.records, sc.desc_pts(),
                                                                            sc.ticket(), sc.totals(), rec, pts, nrm);
        CT_CUDA_CHECK(cudaGetLastError());
        CT_CUDA_CHECK(cudaMemcpyAsync(totals.data() + 2 * i, sc.totals(), 2 * sizeof(unsigned), cudaMemcpyDeviceToHost, stream_));
        CT_CUDA_CHECK(cudaStreamSynchronize(stream_));
    }
    for (size_t i = 0; i < levels_.size(); ++i)
        if (totals[2 * i + 1] != meta.levels[i].num_points)
            throw std::runtime_error("snapshot: the unpacked points of map level " + std::to_string(i) + " disagree with its counters");
    // counters, host copy included: what the saved handle's next frame reads
    MapCounters c[CTICP_MAX_RESOLUTIONS] = {};
    for (size_t i = 0; i < levels_.size(); ++i) {
        const snap::LevelMeta &L = meta.levels[i];
        c[i].num_points = L.num_points;
        c[i].num_voxels = L.num_voxels;
        c[i].num_tombs = L.num_tombs;
        c[i].num_touched = L.num_touched;
        c[i].overflow = L.overflow;
    }
    CT_CUDA_CHECK(cudaMemcpyAsync(d_counters_.data(), c, sizeof(MapCounters) * levels_.size(), cudaMemcpyHostToDevice, stream_));
    memcpy(h_counters_.data(), c, sizeof(MapCounters) * levels_.size());
    frame_count_ = (size_t) meta.frame_count;
    if (with_normals_ && frame_count_) {
        const size_t frames = std::max<size_t>(4096, frame_count_ + 1);
        d_frame_origins_.reserve(3 * frames, stream_);
        CT_CUDA_CHECK(cudaMemcpyAsync(d_frame_origins_.data(), origins, sizeof(double) * 3 * frame_count_, cudaMemcpyDefault, stream_));
    }
    CT_CUDA_CHECK(cudaStreamSynchronize(stream_));
    dirty_ = false;
    readback_pending_ = false;
}

// Pack on this map's stream, copy device to device (a peer copy across devices), unpack on dst's stream
void DeviceMap::CloneInto(DeviceMap &dst, int src_device, int dst_device) {
    CT_CUDA_CHECK(cudaSetDevice(src_device));
    const snap::MapMeta meta = SnapshotMeta();
    const uint64_t bytes = snap::MapSectionBytes(meta) - snap::MapHeaderBytes(meta);
    DeviceArray<unsigned char> packed, copy;
    DeviceArray<double> origins;
    packed.reserve(std::max<uint64_t>(bytes, 16), stream_);
    Pack(packed.data(), meta);   // (synchronises this map's stream)
    CT_CUDA_CHECK(cudaSetDevice(dst_device));
    const size_t n_orig = meta.has_normals ? 3 * (size_t) meta.frame_count : 0;
    copy.reserve(std::max<uint64_t>(bytes, 16), dst.stream_);
    if (n_orig) origins.reserve(n_orig, dst.stream_);
    if (src_device == dst_device) {
        CT_CUDA_CHECK(cudaMemcpyAsync(copy.data(), packed.data(), bytes, cudaMemcpyDeviceToDevice, dst.stream_));
        if (n_orig)
            CT_CUDA_CHECK(cudaMemcpyAsync(origins.data(), d_frame_origins_.data(), sizeof(double) * n_orig, cudaMemcpyDeviceToDevice,
                                          dst.stream_));
    } else {
        // a direct copy over NVLink / PCIe when the GPUs can reach each other; otherwise the driver stages it through host
        // memory
        int can = 0;
        CT_CUDA_CHECK(cudaDeviceCanAccessPeer(&can, dst_device, src_device));
        if (can) {
            const cudaError_t e = cudaDeviceEnablePeerAccess(src_device, 0);
            if (e == cudaErrorPeerAccessAlreadyEnabled) (void) cudaGetLastError();   // (not sticky: clear it)
            else CT_CUDA_CHECK(e);
        }
        CT_CUDA_CHECK(cudaMemcpyPeerAsync(copy.data(), dst_device, packed.data(), src_device, bytes, dst.stream_));
        if (n_orig)
            CT_CUDA_CHECK(cudaMemcpyPeerAsync(origins.data(), dst_device, d_frame_origins_.data(), src_device,
                                              sizeof(double) * n_orig, dst.stream_));
    }
    dst.Unpack(copy.data(), meta, origins.data());   // (synchronises dst's stream: the copies are done)
    copy.clear();
    origins.clear();
    CT_CUDA_CHECK(cudaSetDevice(src_device));
    packed.clear();
}

// ---- Engine -------------------------------------------------------------------------------------------------------------
// Everything already queued on the handle's streams (the speculative map update, the egress) completes first.
void Engine::DrainStreams() {
    CT_CUDA_CHECK(cudaSetDevice(device_));
    CT_CUDA_CHECK(cudaStreamSynchronize(stream_.get()));
    if (aux_stream_.get()) CT_CUDA_CHECK(cudaStreamSynchronize(aux_stream_.get()));
    if (egress_stream_.get()) CT_CUDA_CHECK(cudaStreamSynchronize(egress_stream_.get()));
}

snap::HostState Engine::SnapshotHostState() const {
    snap::HostState s;
    s.registered_frames = registered_frames_;
    s.robust_num_consecutive_failures = robust_num_consecutive_failures_;
    s.next_robust_level = next_robust_level_;
    s.suspect_registration_error = suspect_registration_error_ ? 1 : 0;
    s.cum_distance = tracker_.cum_distance;
    s.cum_orientation = tracker_.cum_orientation;
    s.skipped_frames = tracker_.skipped_frames;
    s.total_insertions = tracker_.total_insertions;
    s.last_num_keypoints = last_num_keypoints_;
    s.prev_frame_points = PrevFramePoints();
    s.default_model_present = default_motion_model_.present ? 1 : 0;
    s.default_model_options = default_motion_model_.options;
    s.default_model_previous_frame = FrameToC(default_motion_model_.previous_frame);
    return s;
}

void Engine::RestoreHostState(const snap::HostState &s, std::vector<HostFrame> trajectory) {
    registered_frames_ = s.registered_frames;
    robust_num_consecutive_failures_ = s.robust_num_consecutive_failures;
    next_robust_level_ = s.next_robust_level;
    suspect_registration_error_ = s.suspect_registration_error != 0;
    tracker_.cum_distance = s.cum_distance;
    tracker_.cum_orientation = s.cum_orientation;
    tracker_.skipped_frames = s.skipped_frames;
    tracker_.total_insertions = s.total_insertions;
    last_num_keypoints_ = (size_t) s.last_num_keypoints;
    restored_prev_frame_points_ = s.prev_frame_points;
    default_motion_model_.present = s.default_model_present != 0;
    default_motion_model_.options = s.default_model_options;
    default_motion_model_.previous_frame = FrameFromC(s.default_model_previous_frame);
    trajectory_ = std::move(trajectory);
}

int64_t Engine::Save(void *dst, size_t cap_bytes) {
    if (shard_world_ > 1) throw UnsupportedError("snapshots of a sharded odometry are not built");
    DrainStreams();
    const snap::MapMeta meta = map_->SnapshotMeta();
    uint64_t size[snap::kNumSections];
    size[snap::kSecOptions] = sizeof(cticp_odometry_options);
    size[snap::kSecHost] = snap::kHostStateBytes;
    size[snap::kSecTrajectory] = 8 + snap::kFrameBytes * trajectory_.size();
    size[snap::kSecMap] = snap::MapSectionBytes(meta);
    size[snap::kSecOrigins] = snap::OriginsBytes(meta);
    const snap::Layout l = snap::MakeLayout(snap::kKindOdometry, size);
    if (!dst) return (int64_t) l.total;
    if (cap_bytes < l.total) throw std::invalid_argument("cticp_odometry_save: cap_bytes below the snapshot size");
    uint8_t *out = static_cast<uint8_t *>(dst);
    snap::WriteHeader(out, l);
    snap::Writer w(out, l.offset[snap::kSecOptions]);
    w.bytes(&options_, sizeof(options_));
    snap::WriteHostState(w, SnapshotHostState());
    w.u64(trajectory_.size());
    for (const HostFrame &f : trajectory_) w.frame(FrameToC(f));
    map_->SaveSection(out + l.offset[snap::kSecMap], out + l.offset[snap::kSecOrigins], meta);
    snap::Seal(out, l);
    return (int64_t) l.total;
}

void DeviceMap::SaveSection(uint8_t *section, uint8_t *origins, const snap::MapMeta &meta) {
    snap::Writer w(section);
    snap::WriteMapHeader(w, meta);
    const uint64_t bytes = snap::MapSectionBytes(meta) - snap::MapHeaderBytes(meta);
    if (bytes) {
        DeviceArray<unsigned char> packed;
        packed.reserve(bytes, stream_);
        Pack(packed.data(), meta);
        CT_CUDA_CHECK(cudaMemcpyAsync(section + snap::MapHeaderBytes(meta), packed.data(), bytes, cudaMemcpyDeviceToHost, stream_));
    }
    if (meta.has_normals && meta.frame_count)
        CT_CUDA_CHECK(cudaMemcpyAsync(origins, d_frame_origins_.data(), 24 * meta.frame_count, cudaMemcpyDeviceToHost, stream_));
    CT_CUDA_CHECK(cudaStreamSynchronize(stream_));
}

void DeviceMap::LoadSection(const snap::Parsed &p) {
    const snap::MapMeta &meta = p.map;
    DeviceArray<unsigned char> payload;
    if (p.map_payload_bytes) {
        payload.reserve(p.map_payload_bytes, stream_);
        CT_CUDA_CHECK(cudaMemcpyAsync(payload.data(), p.base + p.map_payload, p.map_payload_bytes, cudaMemcpyHostToDevice, stream_));
    }
    const double *origins = reinterpret_cast<const double *>(p.base + p.layout.offset[snap::kSecOrigins]);
    Unpack(payload.data(), meta, meta.has_normals ? origins : nullptr);
}

std::unique_ptr<Engine> Engine::Load(const void *src, size_t n_bytes, const cticp_odometry_options *options, int device) {
    snap::Parsed p;
    std::string why;
    if (!snap::Validate(src, n_bytes, snap::kKindOdometry, &p, &why)) throw std::invalid_argument(why);
    cticp_odometry_options saved;
    memcpy(&saved, p.base + p.layout.offset[snap::kSecOptions], sizeof(saved));
    cticp_odometry_options opts = options ? *options : saved;
    if (options) {
        if (!snap::SameMapOptions(options->map_options, saved.map_options))
            throw std::invalid_argument("cticp_odometry_load: options may differ from the saved options only outside map_options");
        if (snap::NeedsNormals(*options) && !p.map.has_normals)
            throw std::invalid_argument("cticp_odometry_load: the options need voxel normals the snapshot does not keep");
    }
    auto e = std::make_unique<Engine>(opts, device);
    snap::Reader h(p.base, p.layout.offset[snap::kSecHost]);
    const snap::HostState s = snap::ReadHostState(h);
    snap::Reader t(p.base, p.layout.offset[snap::kSecTrajectory]);
    std::vector<HostFrame> trajectory(t.u64());
    for (HostFrame &f : trajectory) f = FrameFromC(t.frame());
    e->RestoreHostState(s, std::move(trajectory));
    e->map_->LoadSection(p);
    return e;
}

std::unique_ptr<Engine> Engine::Clone(int device) {
    if (shard_world_ > 1) throw UnsupportedError("clones of a sharded odometry are not built");
    DrainStreams();
    auto e = std::make_unique<Engine>(options_, device);
    e->RestoreHostState(SnapshotHostState(), trajectory_);
    map_->CloneInto(*e->map_, device_, device);
    CT_CUDA_CHECK(cudaSetDevice(device_));
    return e;
}

// ---- standalone maps ------------------------------------------------------------------------------------------------------
int64_t SaveMap(DeviceMap &map, void *dst, size_t cap_bytes) {
    const snap::MapMeta meta = map.SnapshotMeta();
    uint64_t size[snap::kNumSections] = {};
    size[snap::kSecMap] = snap::MapSectionBytes(meta);
    size[snap::kSecOrigins] = snap::OriginsBytes(meta);
    const snap::Layout l = snap::MakeLayout(snap::kKindMap, size);
    if (!dst) return (int64_t) l.total;
    if (cap_bytes < l.total) throw std::invalid_argument("cticp_map_save: cap_bytes below the snapshot size");
    uint8_t *out = static_cast<uint8_t *>(dst);
    snap::WriteHeader(out, l);
    map.SaveSection(out + l.offset[snap::kSecMap], out + l.offset[snap::kSecOrigins], meta);
    snap::Seal(out, l);
    return (int64_t) l.total;
}

void ValidateMapSnapshot(const void *src, size_t n_bytes, snap::Parsed *p) {
    std::string why;
    if (!snap::Validate(src, n_bytes, snap::kKindMap, p, &why)) throw std::invalid_argument(why);
}

}  // namespace cticp
