// neighborhood.h — slam::TNeighborhood (include/SlamCore/experimental/neighborhood.h of the reference) over any point set
// on one device: k-nearest-neighbour search with a bound on the squared distance (NearestNeighborSearchResult +
// SearchNearestNeighbors), and the description of a neighbourhood (ComputeNeighborhood + ComputeNeighborhoodInfo +
// ClassifyNeighborhood), for the k nearest of many queries or for many point sets in one call.
// Semantics, the deviations and the refusals: include/cticp.h, "Neighbourhoods of a point cloud".
#pragma once
#include <cuda_runtime.h>

#include <cstdint>

#include "../../include/cticp.h"
#include "cuda_owner.h"

namespace cticp {

class WorldCloud;

class NeighborhoodIndex {
public:
    static constexpr int kMaxK = 32;                              // one warp lane per neighbour
    static constexpr uint64_t kMaxPoints = (1ull << 31) - 1;      // indices are held in 31 bits on the device
    explicit NeighborhoodIndex(int device);
    ~NeighborhoodIndex();
    NeighborhoodIndex(const NeighborhoodIndex &) = delete;
    NeighborhoodIndex &operator=(const NeighborhoodIndex &) = delete;

    // fp64 xyz triples in host memory, `stride` bytes apart; synchronous
    void BuildHost(const double *xyz, uint64_t stride, uint64_t n);
    // a device scan's xyz (float32 or float64), read after the work queued on `stream`; synchronous
    void BuildDevice(const cticp_device_scan &scan, cudaStream_t stream);
    // the points a world-cloud export returns (index i = export position i), device to device; synchronous
    void BuildWorldCloud(WorldCloud &wc);

    int Device() const { return device_; }
    uint64_t NumPoints() const { return n_; }
    uint64_t NumRejected() const { return rejected_; }
    double CellSize() const { return h_; }

    // m queries (nullptr: the indexed points, m == NumPoints()); host buffers, synchronous
    void Search(const double *queries, uint64_t m, int k, double max_radius, uint64_t *indices, double *d2,
                int32_t *counts);
    void Describe(const double *queries, uint64_t m, int k, double max_radius, int values, double linearity_threshold,
                  double planarity_threshold, cticp_neighborhood_description *out);
    // the same on device buffers of the index's device, ordered after and before `stream`, without a host synchronisation
    void SearchDevice(const double *queries, uint64_t m, int k, double max_radius, uint64_t *indices, double *d2,
                      int32_t *counts, cudaStream_t stream);
    void DescribeDevice(const double *queries, uint64_t m, int k, double max_radius, int values,
                        double linearity_threshold, double planarity_threshold, cticp_neighborhood_description *out,
                        cudaStream_t stream);

    // the argument checks of a search / describe of m queries (std::invalid_argument, UnsupportedError)
    void CheckQuery(const void *queries, uint64_t m, int k, double max_radius) const;

private:
    // ipts_[0, n) holds the points in index order (x, y, z, 0): the cell size, the table and the cell-ordered copy
    void BuildFromIndexed(uint64_t n);
    void Count(double h);   // fills the table at cell size h; occupied_ = the cells used
    void Enqueue(const double *d_queries, uint64_t m, int k, double max_radius, int values, double lin_t,
                 double plan_t, uint64_t *indices, double *d2, int32_t *counts, cticp_neighborhood_description *out,
                 bool describe);

    int device_;
    uint64_t n_ = 0, rejected_ = 0, occupied_ = 0, table_mask_ = 0;
    double lo_[3] = {0, 0, 0}, h_ = 1.0;
    int dims_[3] = {1, 1, 1};
    // the owning members are released in reverse declaration order, after the destructor synchronised the stream
    cticp::Stream stream_;
    Event ev_in_, ev_out_;
    DeviceArray<double4> d_ipts_;          // [n] points in index order
    DeviceArray<double4> d_cpts_;          // [n] valid points by cell: x, y, z, index (bits of a uint64)
    DeviceArray<ulonglong2> d_table_;      // occupied cells: {key, start << 32 | count}, open addressing, linear probing
    DeviceArray<uint32_t> d_fill_;         // [table] points per cell (count pass, then the scatter's cursor)
    DeviceArray<uint32_t> d_pslot_;        // [n] table slot of each point (~0: rejected)
    DeviceArray<double> d_bbox_;           // per-block min / max of the valid points
    DeviceArray<unsigned long long> d_cnt_;   // [0] rejected, [1] occupied cells, [2] points placed
    PinnedArray<unsigned long long> h_cnt_;
    PinnedArray<double> h_bbox_;
    DeviceArray<unsigned char> d_in_;      // host input, as it is
    DeviceArray<double> d_q_;              // host queries
    DeviceArray<uint64_t> d_idx_;
    DeviceArray<double> d_d2_;
    DeviceArray<int32_t> d_counts_;
    DeviceArray<cticp_neighborhood_description> d_desc_;
};

// ComputeNeighborhood(values) + ClassifyNeighborhood(linearity, planarity) of num_sets point sets on `device`: set s is
// points [segment_ends[s - 1], segment_ends[s]) of n fp64 xyz triples in host memory (stride bytes apart)
void DescribePointSets(int device, const double *xyz, uint64_t stride, uint64_t n, const uint64_t *segment_ends,
                       uint64_t num_sets, int values, double linearity_threshold, double planarity_threshold,
                       cticp_neighborhood_description *out);

}  // namespace cticp
