// include/erasor/mapgen.hpp -- ROS-free C++ counterpart of the reference's `class mapgen` (src/mapgen/mapgen.hpp:198-305) on
// top of the C ABI in include/erasor_b200.h (erasor_mapgen_*): the naive map is accumulated on the device, node by node, and
// saveNaiveMap writes the two ASCII PCD files pcl::io::savePCDFileASCII writes, formatted on the device (PcdCodec).
// Everything here goes through the C ABI: no CUDA header or runtime library is needed to use it.
#pragma once
#include <stdexcept>
#include <string>

#include "offline_map_updater.hpp"

namespace erasor_b200 {

class NaiveMapGen {
public:
    // setValue's voxel size and large-scale flag (mapgen.hpp:180-195; main.cpp:87-95)
    explicit NaiveMapGen(float leafsize = 0.05f, bool is_large_scale = false, int device = 0) : device_(device) {
        erasor_mapgen_params_t p{leafsize, is_large_scale ? 1 : 0};
        const int rc = erasor_mapgen_create(&p, device, &g_);
        if (rc == ERASOR_E_INVALID) throw std::invalid_argument(std::string("NaiveMapGen: ") + erasor_mapgen_last_error(nullptr));
        if (rc != ERASOR_OK) throw std::runtime_error(std::string("NaiveMapGen: ") + erasor_mapgen_last_error(nullptr));
    }
    ~NaiveMapGen() { erasor_mapgen_destroy(g_); }
    NaiveMapGen(const NaiveMapGen&) = delete;
    NaiveMapGen& operator=(const NaiveMapGen&) = delete;

    // accumPointCloud(node) (:198-263): odom = {x y z qx qy qz qw} body -> map, lidar in the lidar frame
    void accumPointCloud(const double odom[7], const PointCloud& lidar) {
        check(erasor_mapgen_accum(g_, odom, reinterpret_cast<const float*>(lidar.data()), lidar.size(), ERASOR_PTR_HOST));
    }
    // the same with a scan of n points in device memory (16-byte aligned).  It is read asynchronously: keep it valid and unchanged
    // until the next call that returns data, or until synchronize().
    void accumPointCloud(const double odom[7], const float* lidar_xyzi_device, size_t n) {
        check(erasor_mapgen_accum(g_, odom, lidar_xyzi_device, n, ERASOR_PTR_DEVICE));
    }
    // getPointClouds (:264-268)
    void getPointClouds(PointCloud& map_out, PointCloud& curr_out) {
        map_out = cloud(ERASOR_MAPGEN_CLOUD_MAP);
        curr_out = cloud(ERASOR_MAPGEN_CLOUD_CURR);
    }
    // saveNaiveMap (:270-305): the accumulated map to original_path, the map voxelised at leafsize to map_path
    void saveNaiveMap(const std::string& original_path, const std::string& map_path) {
        PcdCodec codec(device_);
        codec.write(original_path, cloud(ERASOR_MAPGEN_SAVED_ORIGINAL));
        codec.write(map_path, cloud(ERASOR_MAPGEN_SAVED_VOXELIZED));
    }
    // one of the four clouds (ERASOR_MAPGEN_CLOUD_MAP, _CLOUD_CURR, _SAVED_ORIGINAL, _SAVED_VOXELIZED) as a host cloud
    PointCloud cloud(int which) {
        size_t n = 0;
        check(erasor_mapgen_get_cloud(g_, which, nullptr, 0, ERASOR_PTR_HOST, &n));
        PointCloud out(n);
        if (n) check(erasor_mapgen_get_cloud(g_, which, reinterpret_cast<float*>(out.data()), n, ERASOR_PTR_HOST, &n));
        return out;
    }
    void synchronize() { check(erasor_mapgen_synchronize(g_)); }
    erasor_mapgen_t handle() const { return g_; }

private:
    void check(int rc) const {
        if (rc == ERASOR_OK) return;
        const std::string msg = std::string("NaiveMapGen: ") + erasor_mapgen_last_error(g_);
        if (rc == ERASOR_E_INVALID) throw std::invalid_argument(msg);
        throw std::runtime_error(msg);
    }
    erasor_mapgen_t g_ = nullptr;
    int device_ = 0;
};

}  // namespace erasor_b200

// The reference's class is `mapgen` in the global namespace (src/mapgen/mapgen.hpp).  With ERASOR_B200_GLOBAL_NAMES defined,
// code written against it keeps that name.
#ifdef ERASOR_B200_GLOBAL_NAMES
using mapgen = erasor_b200::NaiveMapGen;
#endif
