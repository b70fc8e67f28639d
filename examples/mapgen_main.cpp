// examples/mapgen_main.cpp -- ROS-free counterpart of the reference's kitti_mapgen (src/mapgen/main.cpp): builds the naive map
// from the file layout examples/offline_map_updater_main reads (<data_dir>/poses_lidar2body.csv: a header line, then
// idx,time,x,y,z,qx,qy,qz,qw; <data_dir>/pcds/%06d.pcd, in any PCD DATA mode), node by node on the device (NaiveMapGen), and
// after the last node writes saveNaiveMap's two files under the reference's names (main.cpp:24-35):
//   <save_path>/<seq>_<init>_to_<final>_w_interval<k>_voxel_<std::to_string(voxelsize)>_original.pcd   the accumulated map
//   <save_path>/<seq>_<init>_to_<final>_w_interval<k>_voxel_<std::to_string(voxelsize)>.pcd            ... voxelised at voxelsize
// seq, init, final and k come from the target name, split at '_' as parseRosbagName does (main.cpp:66-101), e.g.
// 05_0_to_2502_w_interval_2_node.bag.
// With a ROS bag of erasor/node messages instead (a path ending in .bag), the nodes are the bag's (NodeBag, as kitti_mapgen receives
// them from rosbag play) and the target name is the bag's file name.
//   usage: mapgen_main <data_dir> <target_name> <save_path> [voxelsize = 0.05] [is_large_scale = false]
//          mapgen_main <file.bag> <save_path> [voxelsize = 0.05] [is_large_scale = false]
#include <cstdio>
#include <cstdlib>
#include <fstream>
#include <iostream>
#include <sstream>

#include <cuda_runtime.h>

#include "../include/erasor/mapgen.hpp"

using namespace erasor_b200;

// A scan in device memory (one float4 per point, 16-byte aligned), grown on demand and reused.
class DeviceCloud {
public:
    DeviceCloud() = default;
    ~DeviceCloud() { if (p_) cudaFree(p_); }
    DeviceCloud(const DeviceCloud&) = delete;
    DeviceCloud& operator=(const DeviceCloud&) = delete;
    float* reserve(size_t n) {
        if (n > cap_ || !p_) {
            if (p_) cudaFree(p_);
            p_ = nullptr; cap_ = 0;
            if (cudaMalloc(reinterpret_cast<void**>(&p_), sizeof(float) * 4 * (n ? n : 1)) != cudaSuccess) throw std::runtime_error("DeviceCloud: cudaMalloc failed");
            cap_ = n;
        }
        return p_;
    }
    const float* data() const { return p_; }
    size_t size() const { return n_; }
    void set_size(size_t n) { n_ = n; }
private:
    float* p_ = nullptr;
    size_t n_ = 0, cap_ = 0;
};

// parseRosbagName (main.cpp:66-79): the '_'-separated tokens before the last '_'
static std::vector<std::string> parse_target_name(std::string name) {
    std::vector<std::string> out;
    size_t pos;
    while ((pos = name.find('_')) != std::string::npos) { out.push_back(name.substr(0, pos)); name.erase(0, pos + 1); }
    return out;
}

// x y z qx qy qz qw per node, parsed as doubles: a file written with 17 significant digits gives back the exact poses
static std::vector<std::array<double, 7>> load_poses(const std::string& csv) {
    std::vector<std::array<double, 7>> poses;
    std::ifstream in(csv);
    if (!in) throw std::invalid_argument("cannot open " + csv);
    std::string line;
    bool first = true;
    while (std::getline(in, line)) {
        if (first) { first = false; continue; }
        std::vector<double> v; std::stringstream ss(line); std::string t;
        while (std::getline(ss, t, ',')) v.push_back(std::stod(t));
        if (v.size() < 9) continue;
        poses.push_back({v[2], v[3], v[4], v[5], v[6], v[7], v[8]});
    }
    return poses;
}

int main(int argc, char** argv) {
    const bool from_bag = argc > 1 && is_bag_path(argv[1]);
    const int a = from_bag ? 1 : 0;                   // the bag form has no target_name argument
    if (argc < 4 - a) {
        std::fprintf(stderr, "usage: %s <data_dir> <target_name> <save_path> [voxelsize = 0.05] [is_large_scale = false]\n"
                             "       %s <file.bag> <save_path> [voxelsize = 0.05] [is_large_scale = false]\n", argv[0], argv[0]);
        return 2;
    }
    try {
        const std::string data_dir = argv[1], save_path = argv[3 - a];
        const std::string target = from_bag ? data_dir.substr(data_dir.find_last_of('/') == std::string::npos ? 0 : data_dir.find_last_of('/') + 1) : argv[2];
        const float voxelsize = argc > 4 - a ? std::stof(argv[4 - a]) : 0.05f;               // /map/voxelsize (main.cpp:87)
        const std::string ls = argc > 5 - a ? argv[5 - a] : "false";                          // /large_scale/is_large_scale (:95)
        const bool is_large_scale = (ls == "true" || ls == "True" || ls == "1");
        const auto parsed = parse_target_name(target);
        if (parsed.size() < 7) throw std::invalid_argument("target name '" + target + "' has fewer than 7 '_'-separated fields before the last");
        const std::string sequence = parsed[0], init_stamp = parsed[1], final_stamp = parsed[3];
        const int interval = std::stoi(parsed[6]);
        const std::string stem = save_path + "/" + sequence + "_" + init_stamp + "_to_" + final_stamp + "_w_interval" + std::to_string(interval) +
                                 "_voxel_" + std::to_string(voxelsize);

        NaiveMapGen gen(voxelsize, is_large_scale);
        if (from_bag) {
            NodeBag bag(data_dir);
            std::cout << "[MAPGEN]: " << bag.size() << " nodes, voxelization size " << voxelsize << ", large-scale " << is_large_scale << std::endl;
            DeviceCloud buf[2];                       // as below: node i + 1 is decoded while node i runs
            auto read = [&](size_t i) { DeviceCloud& b = buf[i % 2]; b.set_size(bag.load_device(i, 1, [&](size_t n) { return b.reserve(n); })[1]); };
            if (bag.size()) read(0);
            for (size_t i = 0; i < bag.size(); ++i) {
                gen.synchronize();
                gen.accumPointCloud(bag.node(i).odom.data(), buf[i % 2].data(), buf[i % 2].size());
                if (i + 1 < bag.size()) read(i + 1);
            }
            gen.saveNaiveMap(stem + "_original.pcd", stem + ".pcd");
            std::cout << "[MAPGEN]: saved " << stem << ".pcd" << std::endl;
            return 0;
        }
        const auto poses = load_poses(data_dir + "/poses_lidar2body.csv");
        std::cout << "[MAPGEN]: " << poses.size() << " nodes, voxelization size " << voxelsize << ", large-scale " << is_large_scale << std::endl;
        PcdCodec codec;
        auto scan_path = [&](size_t i) { char name[64]; std::snprintf(name, sizeof(name), "/pcds/%06zu.pcd", i); return data_dir + name; };
        // Two scan buffers: scan i + 1 is read on the device while node i runs.  The generator reads a device scan asynchronously,
        // so before node i is handed over, node i - 1 -- the last reader of the buffer scan i + 1 will go to -- must be finished.
        DeviceCloud buf[2];
        auto read_scan = [&](size_t i) { DeviceCloud& b = buf[i % 2]; b.set_size(codec.load_device(scan_path(i), [&](size_t n) { return b.reserve(n); })); };
        if (!poses.empty()) read_scan(0);
        for (size_t i = 0; i < poses.size(); ++i) {
            gen.synchronize();
            gen.accumPointCloud(poses[i].data(), buf[i % 2].data(), buf[i % 2].size());
            if (i + 1 < poses.size()) read_scan(i + 1);
        }
        gen.saveNaiveMap(stem + "_original.pcd", stem + ".pcd");
        std::cout << "[MAPGEN]: saved " << stem << ".pcd" << std::endl;
    } catch (const std::exception& e) {
        std::cerr << e.what() << std::endl;
        return 1;
    }
    return 0;
}
