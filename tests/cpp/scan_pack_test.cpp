// Host build of csrc/scan_pack.cuh (plain g++): packs a record buffer the way the engine does and writes every per-point
// output, so that tests/test_device_scan_pack.py can compare it with a NumPy restatement of the format.
//
// usage: scan_pack_test IN OUT n point_step xyz_offset xyz_dtype t_offset t_dtype has_pose begin_ts end_ts
//   IN: n records of point_step bytes. OUT: t_min, t_max (f64), needs_lo (i32), pad (i32), then per point
//   hi[4], lo[4] (f32), the rebuilt x, y, z and timestamp (f64).
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <vector>

#include "scan_pack.cuh"

using namespace cticp::scan_pack;

int main(int argc, char **argv) {
    if (argc != 12) {
        fprintf(stderr, "bad arguments\n");
        return 2;
    }
    const size_t n = strtoull(argv[3], nullptr, 10), step = strtoull(argv[4], nullptr, 10);
    const size_t xoff = strtoull(argv[5], nullptr, 10), toff = strtoull(argv[7], nullptr, 10);
    const int xdt = atoi(argv[6]), tdt = atoi(argv[8]), has_pose = atoi(argv[9]);
    const double bts_arg = strtod(argv[10], nullptr), ets_arg = strtod(argv[11], nullptr);
    std::vector<unsigned char> in(n * step);
    FILE *f = fopen(argv[1], "rb");
    if (!f || fread(in.data(), 1, in.size(), f) != in.size()) return 3;
    fclose(f);
    if (!dtype_size(tdt) || (xdt != 7 && xdt != 8)) return 4;

    double mn = INFINITY, mx = -INFINITY;
    bool any_lo = false;
    std::vector<double> xyz(3 * n), t(n);
    for (size_t i = 0; i < n; ++i) {
        const unsigned char *rec = in.data() + i * step;
        t[i] = decode_timestamp(rec + toff, tdt);
        mn = min_step(mn, t[i]);
        mx = max_step(mx, t[i]);
        for (int k = 0; k < 3; ++k) {
            if (xdt == 7) {
                xyz[3 * i + k] = (double) load_unaligned<float>(rec + xoff + 4 * k);
            } else {
                const double v = load_unaligned<double>(rec + xoff + 8 * k);
                xyz[3 * i + k] = v;
                any_lo = any_lo || needs_lo(v);
            }
        }
    }
    const AlphaRange ar = has_pose ? alpha_range(bts_arg, ets_arg) : alpha_range(mn, mx);
    FILE *o = fopen(argv[2], "wb");
    if (!o) return 5;
    const int32_t head[2] = {any_lo ? 1 : 0, 0};
    fwrite(&mn, 8, 1, o);
    fwrite(&mx, 8, 1, o);
    fwrite(head, 4, 2, o);
    for (size_t i = 0; i < n; ++i) {
        const double a = alpha_of(t[i], ar);
        float hi[4], lo[4];
        for (int k = 0; k < 3; ++k) {
            hi[k] = xdt == 7 ? hi_of((float) xyz[3 * i + k]) : hi_of(xyz[3 * i + k]);
            lo[k] = lo_of(xyz[3 * i + k]);
        }
        hi[3] = hi_of(a);
        lo[3] = lo_of(a);
        double back[4];
        for (int k = 0; k < 3; ++k) back[k] = rebuild(hi[k], lo[k], any_lo);
        back[3] = timestamp_of(hi[3], lo[3], any_lo, ar.mn, ar.mx);
        fwrite(hi, 4, 4, o);
        fwrite(lo, 4, 4, o);
        fwrite(back, 8, 4, o);
    }
    fclose(o);
    printf("SCAN PACK OK\n");
    return 0;
}
