// orc_ply.cpp — dependency-free CPU restatement of the reference's PLY writers and pose reader (src/SlamCore/io.cxx over
// tinyply 2.x), written the way the reference is, not the way the engine is: TEST INFRASTRUCTURE.
//   - WriteCollectionToPLY: one buffer per PLY property, filled item by item with SlamScalarToTinyPLYScalar (a
//     static_cast between the two scalar types), handed to a PlyFile with add_properties_to_element;
//   - the PlyFile keeps its elements in order of first appearance and each property's buffer with a cursor shared by
//     the properties added in one call; write_header streams the header with operator<<, write_binary walks element by
//     element, item by item, property by property, copying each scalar from its buffer at its cursor;
//   - SavePosesAsPLY adds the nine doubles of Float64PosesData and the two ints of pair<int, int> as two calls;
//   - ReadPosesFromPLY parses the header into elements and properties, reads the body, and takes the pose properties by
//     name. Float -> integer out of range or NaN saturates (NaN -> 0): the engine's stated deviation, since the
//     reference's static_cast is undefined there.
#include <cmath>
#include <cstdint>
#include <cstring>
#include <limits>
#include <map>
#include <memory>
#include <sstream>
#include <string>
#include <type_traits>
#include <vector>

namespace {

enum Type { INVALID = 0, INT8 = 1, UINT8, INT16, UINT16, INT32, UINT32, FLOAT32, FLOAT64, INT64, UINT64 };

size_t SizeOf(int t) {
    switch (t) {
        case INT8: case UINT8: return 1;
        case INT16: case UINT16: return 2;
        case INT32: case UINT32: case FLOAT32: return 4;
        case FLOAT64: case INT64: case UINT64: return 8;
        default: return 0;
    }
}

const char *TypeName(int t) {   // tinyply::PropertyTable
    switch (t) {
        case INT8: return "char";
        case UINT8: return "uchar";
        case INT16: return "short";
        case UINT16: return "ushort";
        case INT32: return "int";
        case UINT32: return "uint";
        case FLOAT32: return "float";
        case FLOAT64: return "double";
        default: return "";
    }
}

template <typename To, typename From>
To Cast(From v) {
    if constexpr (std::is_floating_point<From>::value && std::is_integral<To>::value) {
        if (std::isnan(v)) return 0;
        if (!(v > (From) std::numeric_limits<To>::min() - 1)) return std::numeric_limits<To>::min();
        if (!(v < (From) std::numeric_limits<To>::max() + 1)) return std::numeric_limits<To>::max();
    }
    return static_cast<To>(v);
}

template <typename From>
void CastTo(const From &v, char *dst, int to) {
    switch (to) {
        case INT8: { int8_t o = Cast<int8_t>(v); memcpy(dst, &o, 1); break; }
        case UINT8: { uint8_t o = Cast<uint8_t>(v); memcpy(dst, &o, 1); break; }
        case INT16: { int16_t o = Cast<int16_t>(v); memcpy(dst, &o, 2); break; }
        case UINT16: { uint16_t o = Cast<uint16_t>(v); memcpy(dst, &o, 2); break; }
        case INT32: { int32_t o = Cast<int32_t>(v); memcpy(dst, &o, 4); break; }
        case UINT32: { uint32_t o = Cast<uint32_t>(v); memcpy(dst, &o, 4); break; }
        case FLOAT32: { float o = Cast<float>(v); memcpy(dst, &o, 4); break; }
        case FLOAT64: { double o = Cast<double>(v); memcpy(dst, &o, 8); break; }
        default: break;
    }
}

template <typename T>
T Load(const char *p) {
    T v;
    memcpy(&v, p, sizeof(T));
    return v;
}

// SlamScalarToTinyPLYScalar
void ScalarToScalar(const char *src, int from, char *dst, int to) {
    switch (from) {
        case INT8: CastTo(Load<int8_t>(src), dst, to); break;
        case UINT8: CastTo(Load<uint8_t>(src), dst, to); break;
        case INT16: CastTo(Load<int16_t>(src), dst, to); break;
        case UINT16: CastTo(Load<uint16_t>(src), dst, to); break;
        case INT32: CastTo(Load<int32_t>(src), dst, to); break;
        case UINT32: CastTo(Load<uint32_t>(src), dst, to); break;
        case FLOAT32: CastTo(Load<float>(src), dst, to); break;
        case FLOAT64: CastTo(Load<double>(src), dst, to); break;
        case INT64: CastTo(Load<int64_t>(src), dst, to); break;
        case UINT64: CastTo(Load<uint64_t>(src), dst, to); break;
        default: break;
    }
}

// ---- a PlyFile in the manner of tinyply 2.x (writer side) ----------------------------------------------------------
struct PlyData {
    int t = INVALID;
    size_t count = 0;
    const uint8_t *buffer = nullptr;
};
struct Cursor {
    size_t byteOffset = 0;
};
struct Helper {
    std::shared_ptr<PlyData> data;
    std::shared_ptr<Cursor> cursor;
};
struct PlyProperty {
    int t;
    std::string name;
};
struct PlyElement {
    std::string name;
    size_t size;
    std::vector<PlyProperty> properties;
};

class PlyFile {
public:
    void add_properties_to_element(const std::string &element, const std::vector<std::string> &keys, int type,
                                   size_t count, const uint8_t *data) {
        Helper h{std::make_shared<PlyData>(), std::make_shared<Cursor>()};
        h.data->count = count;
        h.data->t = type;
        h.data->buffer = data;
        PlyElement *e = nullptr;
        for (auto &el : elements)
            if (el.name == element) e = &el;
        if (!e) {
            elements.push_back(PlyElement{element, count, {}});
            e = &elements.back();
        }
        for (const auto &k : keys) {
            userData[element + k] = h;
            e->properties.push_back(PlyProperty{type, k});
        }
    }

    void write(std::ostream &os) {
        for (auto &kv : userData) kv.second.cursor->byteOffset = 0;
        write_header(os);
        for (auto &e : elements)
            for (size_t i = 0; i < e.size; ++i)
                for (auto &p : e.properties) {
                    Helper &f = userData[e.name + p.name];
                    const size_t stride = SizeOf(p.t);
                    os.write(reinterpret_cast<const char *>(f.data->buffer) + f.cursor->byteOffset, stride);
                    f.cursor->byteOffset += stride;
                }
    }

private:
    void write_header(std::ostream &os) {
        os << "ply\n";
        os << "format binary_little_endian 1.0" << "\n";
        for (auto &e : elements) {
            os << "element " << e.name << " " << e.size << "\n";
            for (const auto &p : e.properties) os << "property " << TypeName(p.t) << " " << p.name << "\n";
        }
        os << "end_header\n";
    }

    std::vector<PlyElement> elements;
    std::map<std::string, Helper> userData;
};

int64_t Emit(const std::string &s, void *out, uint64_t cap) {
    if (out && cap >= s.size()) memcpy(out, s.data(), s.size());
    return (int64_t) s.size();
}

struct Pose {   // cticp_pose
    double quat[4];
    double tr[3];
    double ref_timestamp, dest_timestamp;
    uint32_t ref_frame_id, dest_frame_id;
};
struct WPoint {   // slam::WPoint3D
    double raw[3];
    double timestamp;
    double world[3];
    uint32_t index_frame, _pad;
};

}  // namespace

extern "C" {

// cticp_ply_property's layout
struct orc_ply_property {
    const char *element;
    const char *name;
    int32_t ply_dtype;
    int32_t src_dtype;
    const void *src;
    uint64_t src_stride_bytes;
};

// WriteCollectionToPLY over a table of columns: returns the size, writes when cap >= size
int64_t orc_ply_write(const orc_ply_property *props, size_t n_props, uint64_t num_items, void *out, uint64_t cap) {
    std::vector<std::vector<uint8_t>> buffers(n_props);
    PlyFile file;
    for (size_t j = 0; j < n_props; ++j) {
        const orc_ply_property &p = props[j];
        const size_t size = SizeOf(p.ply_dtype);
        buffers[j].resize(num_items * size);
        const char *buffer = static_cast<const char *>(p.src);
        for (uint64_t idx = 0; idx < num_items; idx++)
            ScalarToScalar(&buffer[idx * p.src_stride_bytes], p.src_dtype,
                           reinterpret_cast<char *>(&buffers[j][size * idx]), p.ply_dtype);
        file.add_properties_to_element(p.element, {p.name}, p.ply_dtype, num_items, buffers[j].data());
    }
    std::ostringstream os;
    file.write(os);
    return Emit(os.str(), out, cap);
}

// SavePosesAsPLY
int64_t orc_save_poses_ply(const Pose *poses, size_t n, void *out, uint64_t cap) {
    struct Float64PosesData {
        double qs[4];
        double tr[3];
        double ref_t, dest_t;
    };
    std::vector<Float64PosesData> se3(n);
    std::vector<std::pair<int, int>> fids(n);
    for (size_t i = 0; i < n; ++i) {
        const Pose &p = poses[i];
        se3[i] = Float64PosesData{{p.quat[0], p.quat[1], p.quat[2], p.quat[3]}, {p.tr[0], p.tr[1], p.tr[2]},
                                  p.ref_timestamp, p.dest_timestamp};
        fids[i] = std::make_pair(static_cast<int>(p.ref_frame_id), static_cast<int>(p.dest_frame_id));
    }
    PlyFile file;
    file.add_properties_to_element("pose", {"qx", "qy", "qz", "qw", "x", "y", "z", "ref_t", "dest_t"}, FLOAT64, n,
                                   reinterpret_cast<const uint8_t *>(se3.data()));
    file.add_properties_to_element("pose", {"ref_fid", "dest_fid"}, INT32, n,
                                   reinterpret_cast<const uint8_t *>(fids.data()));
    std::ostringstream os;
    file.write(os);
    return Emit(os.str(), out, cap);
}

// WritePLY(os, std::vector<WPoint3D>): BuildDefaultFromSchema(WPoint3D::DefaultSchema()), elements in std::map order,
// a property of dimension d named <name>_<i>
int64_t orc_write_wpoints_ply(const WPoint *pts, size_t n, void *out, uint64_t cap) {
    struct Pty {
        std::string name;
        int type;
        size_t offset;
        int dim;
    };
    std::map<std::string, std::vector<Pty>> schema;   // the element's properties in insertion order
    schema["xyzt"] = {{"xyz", FLOAT64, 0, 3}, {"t", FLOAT64, 24, 1}};
    schema["raw_point"] = {{"x", FLOAT64, 0, 1}, {"y", FLOAT64, 8, 1}, {"z", FLOAT64, 16, 1}};
    schema["world_point"] = {{"x", FLOAT64, 32, 1}, {"y", FLOAT64, 40, 1}, {"z", FLOAT64, 48, 1}};
    schema["properties"] = {{"raw_xyz", FLOAT64, 0, 3}, {"t", FLOAT64, 24, 1}, {"world_xyz", FLOAT64, 32, 3},
                            {"index_frame", UINT32, 56, 1}};
    std::vector<orc_ply_property> props;
    std::vector<std::string> names;
    names.reserve(64);
    for (auto &kv : schema)
        for (auto &p : kv.second)
            for (int d = 0; d < p.dim; ++d) {
                names.push_back(kv.first);
                const char *elem = names.back().c_str();
                names.push_back(p.dim == 1 ? p.name : p.name + "_" + std::to_string(d));
                props.push_back(orc_ply_property{elem, names.back().c_str(), p.type, p.type,
                                                 reinterpret_cast<const char *>(pts) + p.offset + SizeOf(p.type) * d,
                                                 sizeof(WPoint)});
            }
    return orc_ply_write(props.data(), props.size(), n, out, cap);
}

// ReadPosesFromPLY: returns the count (negative for a file the reference rejects), copies min(count, cap)
int64_t orc_read_poses_ply(const void *bytes, size_t n, Pose *out, size_t cap) {
    std::istringstream is(std::string(static_cast<const char *>(bytes), n));
    struct Elem {
        std::string name;
        size_t count;
        std::vector<std::pair<std::string, int>> props;
    };
    std::vector<Elem> elems;
    std::string line;
    if (!std::getline(is, line) || line != "ply") return -1;
    bool little = false;
    while (std::getline(is, line)) {
        std::istringstream ls(line);
        std::string token;
        ls >> token;
        if (token == "end_header") break;
        if (token == "format") {
            std::string fmt;
            ls >> fmt;
            little = fmt == "binary_little_endian";
        } else if (token == "element") {
            Elem e;
            ls >> e.name >> e.count;
            elems.push_back(e);
        } else if (token == "property") {
            std::string type, name;
            ls >> type >> name;
            int t = INVALID;
            for (int k = INT8; k <= FLOAT64; ++k)
                if (type == TypeName(k)) t = k;
            if (t == INVALID || elems.empty()) return -1;
            elems.back().props.emplace_back(name, t);
        } else if (token != "comment" && token != "obj_info") {
            return -1;
        }
    }
    if (!little) return -1;
    const std::string body((std::istreambuf_iterator<char>(is)), std::istreambuf_iterator<char>());
    size_t at = 0;
    static const char *keys[11] = {"qx", "qy", "qz", "qw", "x", "y", "z", "ref_t", "dest_t", "ref_fid", "dest_fid"};
    for (const Elem &e : elems) {
        size_t rec = 0;
        for (auto &p : e.props) rec += SizeOf(p.second);
        if (at + e.count * rec > body.size()) return -1;
        if (e.name != "pose") {
            at += e.count * rec;
            continue;
        }
        size_t off[11];
        for (int k = 0; k < 11; ++k) {
            size_t o = 0;
            bool found = false;
            for (auto &p : e.props) {
                if (p.first == keys[k]) {
                    found = true;
                    if (k < 9 ? p.second != FLOAT64 : (p.second != INT32 && p.second != UINT32)) return -1;
                    break;
                }
                o += SizeOf(p.second);
            }
            if (!found) return -1;
            off[k] = o;
        }
        for (size_t i = 0; i < e.count && i < cap; ++i) {
            const char *r = body.data() + at + i * rec;
            Pose p;
            for (int k = 0; k < 4; ++k) p.quat[k] = Load<double>(r + off[k]);
            for (int k = 0; k < 3; ++k) p.tr[k] = Load<double>(r + off[4 + k]);
            p.ref_timestamp = Load<double>(r + off[7]);
            p.dest_timestamp = Load<double>(r + off[8]);
            p.ref_frame_id = static_cast<uint32_t>(Load<int32_t>(r + off[9]));
            p.dest_frame_id = static_cast<uint32_t>(Load<int32_t>(r + off[10]));
            out[i] = p;
        }
        return (int64_t) e.count;
    }
    return -1;
}

}  // extern "C"
