// ply.cu — see ply.h. Three kernels per call, all on the caller's stream:
//   k_ply_offsets  one CTA: the clamped file ends, each file's size (header + records) and pack-tile count, scanned
//                  into file_offsets and the tile prefix;
//   k_ply_headers  a warp per file: the header from a template built once on the host, the counts formatted here;
//   k_ply_pack     a CTA per tile of consecutive records of one element of one file: columns converted and assembled
//                  in shared memory at the destination's phase mod 16, then written with 16-byte streaming stores.
#include "ply.h"

#include <cctype>
#include <cerrno>
#include <cstdlib>
#include <cstring>
#include <stdexcept>
#include <string>

#include "cuda_owner.h"
#include "device_checks.h"
#include "engine.h"

namespace cticp {
namespace {

constexpr int kMaxProps = 32;
constexpr int kMaxName = 63;
constexpr int kPackThreads = 256;
constexpr int kScanThreads = 1024;
constexpr uint32_t kStageBytes = 32768;   // one pack tile's records: T · max record size <= this
// the longest header without its counts: 32 elements of one property, each name 63 bytes
constexpr int kMaxTemplate = 4 + 32 + 11 + kMaxProps * (8 + kMaxName + 2) + kMaxProps * (9 + 6 + 1 + kMaxName + 1);

struct PlyColumn {
    const unsigned char *src;
    uint64_t stride;
    int32_t sdt, pdt;
    uint32_t rec_off;   // byte offset in its element's record
    uint32_t aligned;   // src and stride are multiples of the source scalar's size
};

struct PlyPlan {
    PlyColumn col[kMaxProps];              // grouped by element, table order within one
    uint32_t elem_first[kMaxProps + 1];    // element e's columns: [elem_first[e], elem_first[e + 1])
    uint32_t rec_size[kMaxProps];
    uint32_t rec_before[kMaxProps];        // record bytes per item of the elements before e
    uint32_t n_elem, rec_total, tmpl_len, tile;
    uint64_t num_items, m, capacity;
};

struct PlyHeader {   // k_ply_headers' parameters: the template travels by value (Hopper takes 32 KB of parameters)
    uint32_t slot[kMaxProps];              // template position where element e's count goes
    uint32_t n_elem, tmpl_len;
    uint64_t m, capacity;
    char tmpl[(kMaxTemplate + 15) / 16 * 16];
};

__constant__ uint64_t c_pow10[20] = {1ull, 10ull, 100ull, 1000ull, 10000ull, 100000ull, 1000000ull, 10000000ull,
                                     100000000ull, 1000000000ull, 10000000000ull, 100000000000ull, 1000000000000ull,
                                     10000000000000ull, 100000000000000ull, 1000000000000000ull,
                                     10000000000000000ull, 100000000000000000ull, 1000000000000000000ull,
                                     10000000000000000000ull};

__host__ __device__ __forceinline__ uint32_t ply_size(int dt) {
    return dt <= 2 ? 1u : dt <= 4 ? 2u : dt <= 7 ? 4u : 8u;   // dt in [1, 10]
}

__device__ __forceinline__ uint32_t num_digits(uint64_t c) {
    uint32_t d = 1;
    while (d < 20 && c >= c_pow10[d]) ++d;
    return d;
}

__device__ __forceinline__ uint64_t load_bits(const unsigned char *p, uint32_t size, bool aligned) {
    if (aligned) {
        switch (size) {
            case 1: return *p;
            case 2: return *reinterpret_cast<const uint16_t *>(p);
            case 4: return *reinterpret_cast<const uint32_t *>(p);
            default: return *reinterpret_cast<const unsigned long long *>(p);
        }
    }
    uint64_t u = 0;   // a misaligned wide load faults: assemble the scalar from bytes
    for (uint32_t b = 0; b < size; ++b) u |= (uint64_t) p[b] << (8 * b);
    return u;
}

// float -> integer: truncation toward zero, saturating at the target's range, NaN -> 0 (the stated deviation)
__device__ __forceinline__ uint64_t saturate_to(double x, int pdt) {
    double lo, hi;
    switch (pdt) {
        case CTICP_DTYPE_INT8: lo = -128.0, hi = 127.0; break;
        case CTICP_DTYPE_UINT8: lo = 0.0, hi = 255.0; break;
        case CTICP_DTYPE_INT16: lo = -32768.0, hi = 32767.0; break;
        case CTICP_DTYPE_UINT16: lo = 0.0, hi = 65535.0; break;
        case CTICP_DTYPE_INT32: lo = -2147483648.0, hi = 2147483647.0; break;
        default: lo = 0.0, hi = 4294967295.0; break;
    }
    if (x != x) return 0;
    const double v = x <= lo ? lo : x >= hi ? hi : x;
    return (uint64_t) (long long) v;   // |v| < 2^32: exact truncation
}

// one scalar: static_cast<ply type>(source value) as g++ on x86-64 computes it; the result's bytes, little-endian
__device__ __forceinline__ uint64_t ply_convert(const unsigned char *p, int sdt, int pdt, bool aligned) {
    const uint64_t raw = load_bits(p, ply_size(sdt), aligned);
    if (sdt == pdt) return raw;
    long long iv = 0;   // integer sources, sign- or zero-extended (UINT64: the raw bits)
    double dv = 0.0;    // float sources
    const bool is_float = sdt == CTICP_DTYPE_FLOAT32 || sdt == CTICP_DTYPE_FLOAT64;
    switch (sdt) {
        case CTICP_DTYPE_INT8: iv = (int8_t) raw; break;
        case CTICP_DTYPE_UINT8: iv = (uint8_t) raw; break;
        case CTICP_DTYPE_INT16: iv = (int16_t) raw; break;
        case CTICP_DTYPE_UINT16: iv = (uint16_t) raw; break;
        case CTICP_DTYPE_INT32: iv = (int32_t) raw; break;
        case CTICP_DTYPE_UINT32: iv = (uint32_t) raw; break;
        case CTICP_DTYPE_FLOAT32: dv = (double) __uint_as_float((uint32_t) raw); break;
        case CTICP_DTYPE_FLOAT64: dv = __longlong_as_double((long long) raw); break;
        default: iv = (long long) raw; break;   // INT64, UINT64
    }
    if (pdt == CTICP_DTYPE_FLOAT32) {
        const float f = is_float ? __double2float_rn(dv)
                                 : sdt == CTICP_DTYPE_UINT64 ? __ull2float_rn(raw) : __ll2float_rn(iv);
        return __float_as_uint(f);
    }
    if (pdt == CTICP_DTYPE_FLOAT64) {
        const double d = is_float ? dv : sdt == CTICP_DTYPE_UINT64 ? __ull2double_rn(raw) : __ll2double_rn(iv);
        return (uint64_t) __double_as_longlong(d);
    }
    return is_float ? saturate_to(dv, pdt) : (uint64_t) iv;   // integer -> integer: the low bytes (modular)
}

// an inclusive block-wide scan (max or sum) of one value per thread over kScanThreads threads, in `s`
template <bool kMax>
__device__ __forceinline__ uint64_t block_scan(uint64_t *s, uint64_t v) {
    s[threadIdx.x] = v;
    __syncthreads();
    for (int d = 1; d < kScanThreads; d <<= 1) {
        const uint64_t o = threadIdx.x >= (unsigned) d ? s[threadIdx.x - d] : 0;
        __syncthreads();
        v = kMax ? (o > v ? o : v) : v + o;
        s[threadIdx.x] = v;
        __syncthreads();
    }
    return v;
}

// Per file k: item_start[k] = the clamped end of file k - 1 (item_start[m] = the last end), file_offsets[k] = the bytes
// of the files before it, tile_prefix[k] = their pack tiles. One CTA walks the files 1024 at a time with carries: the
// offsets are 64-bit sums (tile_lookback carries 32-bit counts) and a call holds thousands of files, not millions.
__global__ void __launch_bounds__(kScanThreads) k_ply_offsets(const PlyPlan P, const uint64_t *__restrict__ file_ends,
                                                              uint64_t *item_start, uint64_t *tile_prefix,
                                                              uint64_t *file_offsets) {
    __shared__ uint64_t s_end[kScanThreads], s_bytes[kScanThreads], s_tiles[kScanThreads];
    uint64_t carry_end = 0, carry_bytes = 0, carry_tiles = 0;
    for (uint64_t base = 0; base < P.m; base += kScanThreads) {
        const uint64_t k = base + threadIdx.x;
        const bool in = k < P.m;
        const uint64_t raw_end = in ? file_ends[k] : 0;
        const uint64_t end_in = block_scan<true>(s_end, raw_end < P.num_items ? raw_end : P.num_items);
        const uint64_t end = end_in > carry_end ? end_in : carry_end;
        uint64_t prev = threadIdx.x ? s_end[threadIdx.x - 1] : 0;
        prev = prev > carry_end ? prev : carry_end;
        const uint64_t c = in ? end - prev : 0;
        const uint64_t bytes = in ? P.tmpl_len + (uint64_t) P.n_elem * num_digits(c) + c * P.rec_total : 0;
        const uint64_t tiles = (c + P.tile - 1) / P.tile;
        const uint64_t bytes_in = block_scan<false>(s_bytes, bytes);
        const uint64_t tiles_in = block_scan<false>(s_tiles, tiles);
        if (in) {
            item_start[k] = prev;
            file_offsets[k] = carry_bytes + bytes_in - bytes;
            tile_prefix[k] = carry_tiles + tiles_in - tiles;
        }
        carry_end = s_end[kScanThreads - 1] > carry_end ? s_end[kScanThreads - 1] : carry_end;
        carry_bytes += s_bytes[kScanThreads - 1];
        carry_tiles += s_tiles[kScanThreads - 1];
        __syncthreads();   // the arrays are rewritten by the next round
    }
    if (threadIdx.x == 0) {
        item_start[P.m] = carry_end;
        file_offsets[P.m] = carry_bytes;
        tile_prefix[P.m] = carry_tiles;
    }
}

// a warp per file: the template with each element's count in decimal at its slot
__global__ void __launch_bounds__(256) k_ply_headers(const __grid_constant__ PlyHeader H,
                                                     const uint64_t *__restrict__ item_start,
                                                     const uint64_t *__restrict__ file_offsets, unsigned char *out) {
    const uint64_t k = ((uint64_t) blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const uint32_t lane = threadIdx.x & 31;
    if (k >= H.m) return;
    const uint64_t c = item_start[k + 1] - item_start[k];
    const uint32_t d = num_digits(c);
    const uint64_t base = file_offsets[k];
    const uint32_t len = H.tmpl_len + H.n_elem * d;
    for (uint32_t i = lane; i < len && base + i < H.capacity; i += 32) {
        char ch = 0;
        bool done = false;
        for (uint32_t e = 0; e < H.n_elem && !done; ++e) {
            if (i < H.slot[e] + e * d) {
                ch = H.tmpl[i - e * d];
                done = true;
            } else if (i < H.slot[e] + (e + 1) * d) {
                ch = (char) ('0' + (c / c_pow10[d - 1 - (i - H.slot[e] - e * d)]) % 10);
                done = true;
            }
        }
        if (!done) ch = H.tmpl[i - H.n_elem * d];
        out[base + i] = (unsigned char) ch;
    }
}

// Tile g of element blockIdx.y: records [r0, r0 + n) of file k, one contiguous destination range. The records are
// assembled at stage[phase + ...], phase = the destination's address mod 16, so stage chunk q is the aligned global
// chunk q of the range: whole chunks go out as 16-byte streaming stores, and only the partial head and tail chunks (the
// ones a neighbouring tile or header shares) as byte stores.
__global__ void __launch_bounds__(kPackThreads) k_ply_pack(const PlyPlan P, const uint64_t *__restrict__ item_start,
                                                           const uint64_t *__restrict__ tile_prefix,
                                                           const uint64_t *__restrict__ file_offsets,
                                                           unsigned char *out) {
    extern __shared__ int4 s_stage4[];
    unsigned char *stage = reinterpret_cast<unsigned char *>(s_stage4);
    __shared__ uint64_t s_k;
    const uint64_t g = blockIdx.x;
    const uint32_t e = blockIdx.y;
    if (g >= tile_prefix[P.m]) return;
    if (threadIdx.x == 0) {   // the last file whose first tile is <= g (empty files share their successor's prefix)
        uint64_t lo = 0, hi = P.m - 1;
        while (lo < hi) {
            const uint64_t mid = (lo + hi + 1) >> 1;
            if (tile_prefix[mid] <= g) lo = mid;
            else hi = mid - 1;
        }
        s_k = lo;
    }
    __syncthreads();
    const uint64_t k = s_k;
    const uint64_t first = item_start[k], c = item_start[k + 1] - first;
    const uint64_t r0 = (g - tile_prefix[k]) * P.tile;
    const uint32_t n = (uint32_t) (c - r0 < P.tile ? c - r0 : P.tile);
    const uint32_t R = P.rec_size[e];
    const uint64_t dst = file_offsets[k] + P.tmpl_len + (uint64_t) P.n_elem * num_digits(c) + c * P.rec_before[e] +
                         r0 * R;
    if (dst >= P.capacity) return;
    const uint64_t end = dst + (uint64_t) n * R < P.capacity ? dst + (uint64_t) n * R : P.capacity;
    const uint32_t phase = (uint32_t) (((uintptr_t) out + dst) & 15);
    const uint32_t c0 = P.elem_first[e], c1 = P.elem_first[e + 1];
    for (uint32_t r = threadIdx.x; r < n; r += kPackThreads) {
        const uint64_t item = first + r0 + r;
        unsigned char *rec = stage + phase + r * R;
        for (uint32_t j = c0; j < c1; ++j) {
            const PlyColumn &C = P.col[j];
            const uint64_t bits = ply_convert(C.src + item * C.stride, C.sdt, C.pdt, C.aligned != 0);
            const uint32_t size = ply_size(C.pdt);
            for (uint32_t b = 0; b < size; ++b) rec[C.rec_off + b] = (unsigned char) (bits >> (8 * b));
        }
    }
    __syncthreads();
    const uint32_t chunks = (uint32_t) ((phase + (end - dst) + 15) / 16);
    unsigned char *a0 = out + dst - phase;   // 16-byte aligned
    for (uint32_t q = threadIdx.x; q < chunks; q += kPackThreads) {
        const uint64_t o = dst - phase + 16ull * q;   // may be below dst only for q = 0
        if (q > 0 || phase == 0) {
            if (o + 16 <= end) {
                __stcs(reinterpret_cast<int4 *>(a0 + 16ull * q), s_stage4[q]);
                continue;
            }
        }
        for (uint32_t b = 0; b < 16; ++b) {
            const uint64_t ob = o + b;
            if ((q > 0 || b >= phase) && ob < end) out[ob] = stage[16 * q + b];
        }
    }
}

const char *PlyTypeName(int dt) {
    static const char *names[] = {"", "char", "uchar", "short", "ushort", "int", "uint", "float", "double"};
    return names[dt];
}

void CheckName(const char *s, const char *what) {
    if (!s) throw std::invalid_argument(std::string(what) + ": null name");
    const size_t n = strnlen(s, kMaxName + 1);
    if (n == 0 || n > (size_t) kMaxName)
        throw std::invalid_argument(std::string(what) + ": names must have 1 to 63 bytes");
    for (size_t i = 0; i < n; ++i)
        if (std::isspace((unsigned char) s[i]))
            throw std::invalid_argument(std::string(what) + " '" + s + "': a name must not contain whitespace");
}

// tinyply 2.x PlyFile::write_header for a binary_little_endian file without comments, as recalled (tinyply is not part
// of this repository): "ply", the format line, per element "element <name> <count>" and its "property <type> <name>"
// lines, "end_header", each ended by '\n'. The counts are left out; slot[e] is where element e's goes.
std::string HeaderTemplate(const std::vector<std::string> &elem_names,
                           const std::vector<std::vector<const cticp_ply_property *>> &elem_props, uint32_t *slot) {
    std::string h = "ply\nformat binary_little_endian 1.0\n";
    for (size_t e = 0; e < elem_names.size(); ++e) {
        h += "element " + elem_names[e] + " ";
        slot[e] = (uint32_t) h.size();
        h += "\n";
        for (const cticp_ply_property *p : elem_props[e])
            h += std::string("property ") + PlyTypeName(p->ply_dtype) + " " + p->name + "\n";
    }
    return h + "end_header\n";
}

struct Plan {
    PlyPlan P{};
    PlyHeader H{};
};

// validates the table and lays it out; src pointers are taken as given (the caller checks or replaces them)
Plan BuildPlan(const cticp_ply_property *props, uint64_t n_props, uint64_t num_items, uint64_t m, uint64_t capacity) {
    if (!props) throw std::invalid_argument("null properties");
    if (n_props == 0 || n_props > (uint64_t) kMaxProps) throw std::invalid_argument("n_props must be in [1, 32]");
    std::vector<std::string> names;
    std::vector<std::vector<const cticp_ply_property *>> groups;
    for (uint64_t i = 0; i < n_props; ++i) {
        const cticp_ply_property &p = props[i];
        CheckName(p.element, "element");
        CheckName(p.name, "property");
        if (p.ply_dtype < CTICP_DTYPE_INT8 || p.ply_dtype > CTICP_DTYPE_FLOAT64)
            throw std::invalid_argument(std::string("property ") + p.name + ": unknown ply_dtype");
        if (p.src_dtype < CTICP_DTYPE_INT8 || p.src_dtype > CTICP_DTYPE_UINT64)
            throw std::invalid_argument(std::string("property ") + p.name + ": unknown src_dtype");
        if (!p.src && num_items) throw std::invalid_argument(std::string("property ") + p.name + ": null source");
        size_t e = 0;
        while (e < names.size() && names[e] != p.element) ++e;
        if (e == names.size()) {
            names.emplace_back(p.element);
            groups.emplace_back();
        }
        for (const cticp_ply_property *q : groups[e])
            if (strcmp(q->name, p.name) == 0)
                throw std::invalid_argument(std::string("property ") + p.name + " appears twice in element " +
                                            p.element);
        groups[e].push_back(&p);
    }
    Plan plan;
    PlyPlan &P = plan.P;
    P.n_elem = (uint32_t) names.size();
    uint32_t j = 0, rmax = 0;
    for (uint32_t e = 0; e < P.n_elem; ++e) {
        P.elem_first[e] = j;
        P.rec_before[e] = P.rec_total;
        uint32_t off = 0;
        for (const cticp_ply_property *p : groups[e]) {
            P.col[j++] = PlyColumn{static_cast<const unsigned char *>(p->src), p->src_stride_bytes, p->src_dtype,
                                   p->ply_dtype, off, 0};
            off += ply_size(p->ply_dtype);
        }
        P.rec_size[e] = off;
        P.rec_total += off;
        rmax = off > rmax ? off : rmax;
    }
    P.elem_first[P.n_elem] = j;
    P.tile = 2048;
    while (P.tile > 128 && P.tile * rmax > kStageBytes) P.tile >>= 1;
    P.num_items = num_items;
    P.m = m;
    P.capacity = capacity;
    const std::string t = HeaderTemplate(names, groups, plan.H.slot);
    if (t.size() > sizeof(plan.H.tmpl)) throw std::logic_error("PLY header template overflow");
    memcpy(plan.H.tmpl, t.data(), t.size());
    P.tmpl_len = plan.H.tmpl_len = (uint32_t) t.size();
    plan.H.n_elem = P.n_elem;
    plan.H.m = m;
    plan.H.capacity = capacity;
    return plan;
}

uint64_t HostDigits(uint64_t c) {
    uint64_t d = 1;
    while (c >= 10) c /= 10, ++d;
    return d;
}

// the three kernels on `stream`; the columns' src pointers are device memory of the current device
void Enqueue(Plan &plan, const uint64_t *file_ends, unsigned char *out, uint64_t *file_offsets, cudaStream_t stream) {
    PlyPlan &P = plan.P;
    for (uint32_t j = 0; j < P.elem_first[P.n_elem]; ++j) {
        PlyColumn &C = P.col[j];
        const uint64_t size = ply_size(C.sdt);
        C.aligned = ((uintptr_t) C.src % size == 0 && C.stride % size == 0) ? 1u : 0u;
    }
    const uint64_t pack_x = (P.num_items + P.tile - 1) / P.tile + P.m;
    if (pack_x > 0x7fffffffull) throw std::invalid_argument("too many items and files for one call");
    void *scratch = nullptr;
    CT_CUDA_CHECK(cudaMallocAsync(&scratch, sizeof(uint64_t) * 2 * (P.m + 1), stream));
    uint64_t *item_start = static_cast<uint64_t *>(scratch), *tile_prefix = item_start + P.m + 1;
    k_ply_offsets<<<1, kScanThreads, 0, stream>>>(P, file_ends, item_start, tile_prefix, file_offsets);
    if (P.capacity && P.m) {
        k_ply_headers<<<(unsigned) ((P.m * 32 + 255) / 256), 256, 0, stream>>>(plan.H, item_start, file_offsets, out);
        if (P.num_items) {
            uint32_t rmax = 0;
            for (uint32_t e = 0; e < P.n_elem; ++e) rmax = P.rec_size[e] > rmax ? P.rec_size[e] : rmax;
            const size_t smem = (16 + (size_t) P.tile * rmax + 15) / 16 * 16;
            k_ply_pack<<<dim3((unsigned) pack_x, P.n_elem), kPackThreads, smem, stream>>>(P, item_start, tile_prefix,
                                                                                      file_offsets, out);
        }
    }
    CT_CUDA_CHECK(cudaGetLastError());
    CT_CUDA_CHECK(cudaFreeAsync(scratch, stream));
}

void RequireAligned8(const void *p, const char *what) {
    if ((uintptr_t) p % 8) throw std::invalid_argument(std::string(what) + ": must be 8-byte aligned");
}

}  // namespace

void PlyWriteDevice(int device, const cticp_ply_property *props, uint64_t n_props, uint64_t num_items,
                    const uint64_t *file_ends, uint64_t m, void *out, uint64_t capacity, uint64_t *file_offsets,
                    cudaStream_t stream) {
    Plan plan = BuildPlan(props, n_props, num_items, m, capacity);
    if ((m && !file_ends) || !file_offsets || (capacity && !out)) throw std::invalid_argument("null argument");
    CT_CUDA_CHECK(cudaSetDevice(device));
    if (num_items) {
        for (uint64_t i = 0; i < n_props; ++i) {
            const std::string what = std::string("property ") + props[i].name;
            RequireDeviceRange(props[i].src,
                               SpanBytes(num_items, props[i].src_stride_bytes, ply_size(props[i].src_dtype),
                                         what.c_str()),
                               device, what.c_str());
        }
    }
    if (m) {
        RequireAligned8(file_ends, "file_ends");
        RequireDeviceRange(file_ends, 8 * m, device, "file_ends");
    }
    RequireAligned8(file_offsets, "file_offsets");
    RequireDeviceRange(file_offsets, 8 * (m + 1), device, "file_offsets");
    if (capacity) RequireDeviceRange(out, capacity, device, "out");
    Enqueue(plan, file_ends, static_cast<unsigned char *>(out), file_offsets, stream);
}

uint64_t PlyWrite(int device, const cticp_ply_property *props, uint64_t n_props, uint64_t num_items, void *out,
                  uint64_t capacity) {
    Plan plan = BuildPlan(props, n_props, num_items, 1, capacity);
    PlyPlan &P = plan.P;
    const uint64_t size = P.tmpl_len + P.n_elem * HostDigits(num_items) + num_items * P.rec_total;
    if (capacity < size) return size;
    if (!out) throw std::invalid_argument("null argument");
    CT_CUDA_CHECK(cudaSetDevice(device));
    Stream stream(cudaStreamNonBlocking);
    const cudaStream_t s = stream.get();
    // the columns side by side, each at a 16-byte boundary plus its own address's phase (so its alignment is kept)
    const uint32_t n_cols = P.elem_first[P.n_elem];
    std::vector<uint64_t> at(n_cols), span(n_cols);
    uint64_t total = 8 * 3;   // file_ends[1], file_offsets[2]
    for (uint32_t j = 0; j < n_cols; ++j) {
        span[j] = num_items ? SpanBytes(num_items, P.col[j].stride, ply_size(P.col[j].sdt), "property") : 0;
        at[j] = (total + 15) / 16 * 16 + ((uintptr_t) P.col[j].src & 15);
        total = at[j] + span[j];
    }
    DeviceArray<unsigned char> d_cols, d_out;
    d_cols.reserve(total, s);
    d_out.reserve(size, s);
    uint64_t *d_ends = reinterpret_cast<uint64_t *>(d_cols.data()), *d_offsets = d_ends + 1;
    CT_CUDA_CHECK(cudaMemcpyAsync(d_ends, &num_items, 8, cudaMemcpyHostToDevice, s));
    for (uint32_t j = 0; j < n_cols; ++j) {
        if (span[j])
            CT_CUDA_CHECK(cudaMemcpyAsync(d_cols.data() + at[j], P.col[j].src, span[j], cudaMemcpyHostToDevice, s));
        P.col[j].src = d_cols.data() + at[j];
    }
    P.capacity = plan.H.capacity = size;
    Enqueue(plan, d_ends, d_out.data(), d_offsets, s);
    CT_CUDA_CHECK(cudaMemcpyAsync(out, d_out.data(), size, cudaMemcpyDeviceToHost, s));
    CT_CUDA_CHECK(cudaStreamSynchronize(s));
    return size;
}

// ---- pose files ----------------------------------------------------------------------------------------------------
std::vector<cticp_pose> PlyReadPoses(const char *bytes, uint64_t n) {
    if (!bytes) throw std::invalid_argument("null argument");
    struct Prop {
        std::string name;
        int dtype;
        uint32_t offset;
    };
    struct Elem {
        std::string name;
        uint64_t count;
        uint32_t rec = 0;
        std::vector<Prop> props;
    };
    std::vector<Elem> elems;
    uint64_t pos = 0;
    bool format = false;
    auto words = [](const std::string &line) {
        std::vector<std::string> w;
        size_t i = 0;
        while (i < line.size()) {
            while (i < line.size() && std::isspace((unsigned char) line[i])) ++i;
            size_t j = i;
            while (j < line.size() && !std::isspace((unsigned char) line[j])) ++j;
            if (j > i) w.push_back(line.substr(i, j - i));
            i = j;
        }
        return w;
    };
    auto type_of = [](const std::string &t) {
        static const char *a[] = {"", "char", "uchar", "short", "ushort", "int", "uint", "float", "double"};
        static const char *b[] = {"", "int8", "uint8", "int16", "uint16", "int32", "uint32", "float32", "float64"};
        for (int d = 1; d <= 8; ++d)
            if (t == a[d] || t == b[d]) return d;
        return 0;
    };
    for (bool first = true;; first = false) {
        const void *nl = pos < n ? memchr(bytes + pos, '\n', n - pos) : nullptr;
        if (!nl) throw std::invalid_argument("PLY: the header has no end_header line");
        const uint64_t e = static_cast<const char *>(nl) - bytes;
        const std::vector<std::string> w = words(std::string(bytes + pos, e - pos));
        pos = e + 1;
        if (first) {
            if (w != std::vector<std::string>{"ply"}) throw std::invalid_argument("PLY: no ply magic");
            continue;
        }
        if (w.empty() || w[0] == "comment" || w[0] == "obj_info") continue;
        if (w[0] == "end_header") break;
        if (w[0] == "format") {
            if (w.size() < 2) throw std::invalid_argument("PLY: a malformed format line");
            if (w[1] == "ascii" || w[1] == "binary_big_endian")
                throw UnsupportedError("PLY: " + w[1] + " bodies are not supported (binary_little_endian only)");
            if (w[1] != "binary_little_endian") throw std::invalid_argument("PLY: unknown format " + w[1]);
            format = true;
        } else if (w[0] == "element") {
            if (w.size() != 3 || w[2].empty() || w[2][0] == '-') throw std::invalid_argument("PLY: a malformed element line");
            char *end = nullptr;
            errno = 0;
            const uint64_t count = std::strtoull(w[2].c_str(), &end, 10);
            if (errno || *end) throw std::invalid_argument("PLY: a malformed element count");
            elems.push_back(Elem{w[1], count});
        } else if (w[0] == "property") {
            if (elems.empty()) throw std::invalid_argument("PLY: a property outside an element");
            if (w.size() >= 2 && w[1] == "list") throw UnsupportedError("PLY: list properties are not supported");
            if (w.size() != 3) throw std::invalid_argument("PLY: a malformed property line");
            const int dt = type_of(w[1]);
            if (!dt) throw std::invalid_argument("PLY: unknown property type " + w[1]);
            Elem &el = elems.back();
            el.props.push_back(Prop{w[2], dt, el.rec});
            el.rec += ply_size(dt);
        } else {
            throw std::invalid_argument("PLY: unknown header line");
        }
    }
    if (!format) throw std::invalid_argument("PLY: no format line");
    uint64_t body = pos;
    const Elem *pose = nullptr;
    uint64_t pose_at = 0;
    for (const Elem &el : elems) {
        uint64_t bytes_of = 0;
        if (__builtin_mul_overflow(el.count, (uint64_t) el.rec, &bytes_of) ||
            __builtin_add_overflow(body, bytes_of, &body))
            throw std::invalid_argument("PLY: the body is shorter than the header says");
        if (el.name == "pose" && !pose) pose = &el, pose_at = body - bytes_of;
    }
    if (body > n) throw std::invalid_argument("PLY: the body is shorter than the header says");
    if (!pose) throw std::invalid_argument("PLY: no pose element");
    static const char *names[11] = {"qx", "qy", "qz", "qw", "x", "y", "z", "ref_t", "dest_t", "ref_fid", "dest_fid"};
    uint32_t off[11];
    for (int i = 0; i < 11; ++i) {
        const Prop *p = nullptr;
        for (const Prop &q : pose->props)
            if (q.name == names[i]) p = &q;
        if (!p) throw std::invalid_argument(std::string("PLY: the pose element has no property ") + names[i]);
        if (i < 9 && p->dtype != CTICP_DTYPE_FLOAT64)
            throw std::invalid_argument("PLY: invalid types in the poses file (expected float64)");
        if (i >= 9 && p->dtype != CTICP_DTYPE_INT32 && p->dtype != CTICP_DTYPE_UINT32)
            throw std::invalid_argument("PLY: the frame ids must be int or uint");
        off[i] = p->offset;
    }
    std::vector<cticp_pose> out(pose->count);
    for (uint64_t k = 0; k < pose->count; ++k) {
        const char *rec = bytes + pose_at + k * pose->rec;
        double v[9];
        for (int i = 0; i < 9; ++i) memcpy(&v[i], rec + off[i], 8);
        cticp_pose &p = out[k];
        memcpy(p.quat, v, 32);
        memcpy(p.tr, v + 4, 24);
        p.ref_timestamp = v[7];
        p.dest_timestamp = v[8];
        memcpy(&p.ref_frame_id, rec + off[9], 4);
        memcpy(&p.dest_frame_id, rec + off[10], 4);
    }
    return out;
}

}  // namespace cticp
