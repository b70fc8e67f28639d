// examples/offline_map_updater_main.cpp -- ROS-free counterpart of the reference's file-based driver
// src/offline_map_updater/main_in_your_env.cpp:60-127: reads <data_dir>/dense_global_map.pcd,
// <data_dir>/poses_lidar2body.csv (header line, then  idx,time,x,y,z,qx,qy,qz,qw ; columns 2..8 are used, :46-49)
// and <data_dir>/pcds/%06d.pcd (each read on the device by PcdCodec::load, in any DATA mode: ascii, binary or binary_compressed, as
// the reference's pcl::io::loadPCDFile reads them), feeds every node to the device-resident OfflineMapUpdater and writes
// <save_path>/<data_name>_result.pcd with save_static_map(0.2) (:123), formatted on the device.
// With a path ending in .bag instead of <data_dir>, the nodes come from a ROS bag of erasor/node messages (NodeBag, as the reference's
// offline_map_updater receives them from rosbag play): the map is the yaml's initial_map_path, read by PcdCodec::load; seq is each
// node's header.seq and its odom goes in as the bag's doubles; each next cloud is decoded on the device into the second buffer.
//   usage: offline_map_updater_main <config.yaml> <data_dir> [init_idx]
//          offline_map_updater_main <config.yaml> <file.bag> [init_idx]
#include <cstdio>
#include <cstdlib>
#include <fstream>
#include <iostream>
#include <sstream>

#include <cuda_runtime.h>

#include "../include/erasor/offline_map_updater.hpp"

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
    void swap(DeviceCloud& o) { std::swap(p_, o.p_); std::swap(n_, o.n_); std::swap(cap_, o.cap_); }
private:
    float* p_ = nullptr;
    size_t n_ = 0, cap_ = 0;
};

// The scan is read on the device straight into `out`, complete on return.
static void read_scan(PcdCodec& codec, const std::string& path, DeviceCloud& out) {
    out.set_size(codec.load_device(path, [&](size_t n) { return out.reserve(n); }));
}

static std::vector<std::array<double, 7>> load_all_poses(const std::string& txt) {
    std::vector<std::array<double, 7>> poses;
    std::ifstream in(txt);
    if (!in) throw std::invalid_argument("cannot open " + txt);
    std::string line;
    bool first = true;
    while (std::getline(in, line)) {
        if (first) { first = false; continue; }
        std::vector<float> v; std::stringstream ss(line); std::string t;
        while (std::getline(ss, t, ',')) v.push_back(std::stof(t));
        if (v.size() < 9) continue;
        // the reference builds Eigen::Quaternionf(w=pose[8], x=pose[5], y=pose[6], z=pose[7]) and a float translation (:46-47)
        poses.push_back({v[2], v[3], v[4], v[5], v[6], v[7], v[8]});
    }
    std::cout << "Total " << poses.size() << " poses are loaded" << std::endl;
    return poses;
}

// the bag form: the same loop over the bag's nodes
static void run_bag(const Config& cfg, const std::string& bag_path, int init_idx) {
    PcdCodec codec;
    PointCloud map = codec.load(cfg.initial_map_path);
    OfflineMapUpdater updater(cfg, map);
    PointCloud().swap(map);
    NodeBag bag(bag_path);
    std::cout << "Total " << bag.size() << " nodes are loaded" << std::endl;
    auto read = [&](size_t i, DeviceCloud& out) { out.set_size(bag.load_device(i, 1, [&](size_t n) { return out.reserve(n); })[1]); };
    const size_t n_nodes = bag.size(), first = init_idx > 0 ? (size_t)init_idx : 0;
    DeviceCloud cur, nxt;
    if (first < n_nodes) read(first, cur);
    for (size_t i = first; i < n_nodes; ++i) {
        if (i + 1 < n_nodes) {
            read(i + 1, nxt);
            if (updater.processes_call(2)) updater.prefetch_device(nxt.data(), nxt.size());
        }
        updater.callback_node_device((int)bag.node(i).seq, bag.node(i).odom.data(), cur.data(), cur.size());
        cur.swap(nxt);
    }
    updater.save_static_map(0.2f);
    std::cout << "Static map building complete!" << std::endl;
}

int main(int argc, char** argv) {
    if (argc < 3) { std::fprintf(stderr, "usage: %s <config.yaml> <data_dir | file.bag> [init_idx]\n", argv[0]); return 2; }
    try {
        Config cfg = load_config(argv[1]);
        const std::string data_dir = argv[2];
        const int init_idx = argc > 3 ? std::atoi(argv[3]) : 0;
        if (is_bag_path(data_dir)) { run_bag(cfg, data_dir, init_idx); return 0; }
        cfg.initial_map_path = data_dir + "/dense_global_map.pcd";
        PcdCodec codec;
        PointCloud map = codec.load(cfg.initial_map_path);
        OfflineMapUpdater updater(cfg, map);
        PointCloud().swap(map);
        const auto poses = load_all_poses(data_dir + "/poses_lidar2body.csv");
        // Scans come from files, so the next one is known: it is read on the device (into device memory, complete when
        // load_device returns) before the current node is processed and, when that next call will process its node
        // (removal_interval), handed to the updater's look-ahead -- its voxelisation then runs under the current node's path.
        auto scan_path = [&](int i) { char name[64]; std::snprintf(name, sizeof(name), "/pcds/%06d.pcd", i); return data_dir + name; };
        const int n_nodes = (int)poses.size();
        DeviceCloud cur, nxt;
        if (init_idx < n_nodes) read_scan(codec, scan_path(init_idx), cur);
        for (int i = init_idx; i < n_nodes; ++i) {
            if (i + 1 < n_nodes) {
                read_scan(codec, scan_path(i + 1), nxt);
                if (updater.processes_call(2)) updater.prefetch_device(nxt.data(), nxt.size());
            }
            updater.callback_node_device(i, poses[i].data(), cur.data(), cur.size());
            cur.swap(nxt);
        }
        updater.save_static_map(0.2f);
        std::cout << "Static map building complete!" << std::endl;
    } catch (const std::exception& e) {
        std::cerr << e.what() << std::endl;
        return 1;
    }
    return 0;
}
