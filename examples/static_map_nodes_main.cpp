// examples/static_map_nodes_main.cpp -- the frame-independent twin of offline_map_updater_main: the same file layout
// (<data_dir>/dense_global_map.pcd, <data_dir>/poses_lidar2body.csv, <data_dir>/pcds/%06d.pcd) and the same config yaml, but every
// node that callback_node would process (every removal_interval-th call) is tested against the same initial map in node mode
// (erasor_process_nodes), in batches.  The map and every scan are read on the device by PcdCodec::load_device, in any DATA mode; a
// batch's raw scans are voxelised and moved to the body frame on the device in one submission (ERASOR::process_scans).  The kept
// map, voxelised at 0.2 m as offline_map_updater_main saves it (main_in_your_env.cpp:123), goes to <save_path>/<data_name>_result.pcd,
// formatted on the device.  One GPU; multi-GPU callers shard the nodes and combine the masks with erasor_comm_*.
// With a ROS bag of erasor/node messages instead of <data_dir> (a path ending in .bag), the map is the yaml's initial_map_path, the
// poses are the bag's doubles, and each batch's clouds are decoded from the bag on the device in one call (NodeBag::load_device).
// inserts = 1 turns node-mode inserts on: the query points each node's static estimate puts back into the map are saved with it.
// inserts = 2 also re-tests them (DESIGN.md section 8.4.1): a second pass over the same batches against the kept map followed by
// every node's inserts, each node seeing the inserts of the nodes before it; the re-test map under that pass's mask is saved.
//   usage: static_map_nodes_main <config.yaml> <data_dir> [init_idx] [batch] [inserts]
//          static_map_nodes_main <config.yaml> <file.bag> [init_idx] [batch] [inserts]
#include <cstdio>
#include <cstdlib>
#include <fstream>
#include <iostream>
#include <sstream>

#include <cuda_runtime.h>

#include "../include/erasor/offline_map_updater.hpp"

using namespace erasor_b200;

// device memory owned here (16-byte aligned: cudaMalloc); growing keeps the first `keep` points
class DeviceBuffer {
public:
    DeviceBuffer() = default;
    ~DeviceBuffer() { if (p_) cudaFree(p_); }
    DeviceBuffer(const DeviceBuffer&) = delete;
    DeviceBuffer& operator=(const DeviceBuffer&) = delete;
    float* reserve(size_t n_points, size_t keep = 0) {
        if (n_points > cap_ || !p_) {
            const size_t cap = std::max<size_t>({n_points, 2 * cap_, 1});
            float* q = nullptr;
            if (cudaMalloc(reinterpret_cast<void**>(&q), sizeof(float) * 4 * cap) != cudaSuccess) throw std::runtime_error("DeviceBuffer: cudaMalloc failed");
            if (keep && (cudaMemcpy(q, p_, sizeof(float) * 4 * keep, cudaMemcpyDeviceToDevice) != cudaSuccess || cudaDeviceSynchronize() != cudaSuccess))
                throw std::runtime_error("DeviceBuffer: copy failed");
            if (p_) cudaFree(p_);
            p_ = q; cap_ = cap;
        }
        return p_;
    }
    float* data() const { return p_; }
private:
    float* p_ = nullptr;
    size_t cap_ = 0;
};

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
        poses.push_back({v[2], v[3], v[4], v[5], v[6], v[7], v[8]});   // as main_in_your_env.cpp:46-47 reads them (floats)
    }
    std::cout << "Total " << poses.size() << " poses are loaded" << std::endl;
    return poses;
}

int main(int argc, char** argv) {
    if (argc < 3) { std::fprintf(stderr, "usage: %s <config.yaml> <data_dir> [init_idx] [batch] [inserts]\n", argv[0]); return 2; }
    try {
        Config cfg = load_config(argv[1]);
        const std::string data_dir = argv[2];
        const int init_idx = argc > 3 ? std::atoi(argv[3]) : 0;
        const int batch = argc > 4 ? std::max(1, std::atoi(argv[4])) : 20;
        const int inserts_arg = argc > 5 ? std::atoi(argv[5]) : 0;
        if (inserts_arg < 0 || inserts_arg > 2) throw std::invalid_argument("inserts must be 0 (off), 1 (on) or 2 (on, with the re-test pass)");
        const bool inserts = inserts_arg != 0, retest = inserts_arg == 2;
        if (cfg.updater.is_large_scale) throw std::invalid_argument("node mode has no large-scale windowing: use offline_map_updater_main");
        if (cfg.updater.removal_interval < 1) throw std::invalid_argument("removal_interval must be >= 1");
        erasor_params_t ep = cfg.erasor;
        ep.version = cfg.updater.version;                               // /erasor/version as the updater reads it (:81)
        ERASOR erasor(ep);
        erasor.set_node_inserts(inserts);
        PcdCodec codec;
        DeviceBuffer map;
        const bool from_bag = is_bag_path(data_dir);
        const size_t n_map = codec.load_device(from_bag ? cfg.initial_map_path : data_dir + "/dense_global_map.pcd", [&](size_t n) { return map.reserve(n); });
        erasor.load_global_map_device(map.data(), n_map);
        std::array<double, 7> l2b;
        for (int i = 0; i < 7; ++i) l2b[i] = cfg.updater.lidar2body[i];
        if (from_bag) {
            NodeBag bag(data_dir);
            std::vector<uint64_t> sel;
            for (size_t i = init_idx > 0 ? (size_t)init_idx : 0; i < bag.size(); ++i)
                if ((i - init_idx + 1) % cfg.updater.removal_interval == 0) sel.push_back(i);
            DeviceBuffer raw;
            for (int pass = 0; pass < (retest ? 2 : 1); ++pass) {
                if (pass == 1) erasor.begin_retest();
                for (size_t b0 = 0; b0 < sel.size(); b0 += (size_t)batch) {
                    const std::vector<uint64_t> nodes(sel.begin() + b0, sel.begin() + std::min(sel.size(), b0 + (size_t)batch));
                    std::vector<std::array<double, 7>> bp;
                    for (uint64_t i : nodes) bp.push_back(bag.node(i).odom);
                    const std::vector<uint64_t> off = bag.load_device(nodes, [&](size_t m) { return raw.reserve(m); });
                    if (pass == 0) erasor.process_scans(bp, raw.data(), off, cfg.updater.query_voxel_size, l2b, cfg.updater.max_range, ERASOR_PTR_DEVICE);
                    else erasor.process_scans_retest(bp, raw.data(), off, (int)b0, cfg.updater.query_voxel_size, l2b, cfg.updater.max_range, ERASOR_PTR_DEVICE);
                }
            }
            const ERASOR::DeviceClouds saved = erasor.save_static_map(0.2f);
            const std::string target = cfg.save_path + "/" + cfg.data_name + "_result.pcd";
            codec.write_device(target, saved.d_xyzi, saved.offsets[1]);
            std::cout << sel.size() << " of " << bag.size() << " bag nodes processed; " << saved.offsets[1] << " points saved to " << target << std::endl;
            return 0;
        }
        const auto poses = load_all_poses(data_dir + "/poses_lidar2body.csv");
        // the nodes callback_node processes: its k-th call (k = 1, 2, ...) unless k % removal_interval != 0 ("PASS!", :328)
        std::vector<int> sel;
        for (int i = init_idx; i < (int)poses.size(); ++i)
            if ((i - init_idx + 1) % cfg.updater.removal_interval == 0) sel.push_back(i);
        auto scan_path = [&](int i) { char name[64]; std::snprintf(name, sizeof(name), "/pcds/%06d.pcd", i); return data_dir + name; };
        DeviceBuffer raw;                                               // a batch's raw scans, back to back
        for (int pass = 0; pass < (retest ? 2 : 1); ++pass) {
            if (pass == 1) erasor.begin_retest();                       // the re-test pass reads the same scans again
            for (size_t b0 = 0; b0 < sel.size(); b0 += (size_t)batch) {
                const size_t nb = std::min(sel.size() - b0, (size_t)batch);
                std::vector<std::array<double, 7>> bp(nb);
                std::vector<uint64_t> off(nb + 1, 0);
                for (size_t j = 0; j < nb; ++j) {                       // each scan read on the device behind the previous one
                    bp[j] = poses[sel[b0 + j]];
                    off[j + 1] = off[j] + codec.load_device(scan_path(sel[b0 + j]), [&](size_t m) { return raw.reserve(off[j] + m, off[j]) + 4 * off[j]; });
                }
                if (pass == 0) erasor.process_scans(bp, raw.data(), off, cfg.updater.query_voxel_size, l2b, cfg.updater.max_range, ERASOR_PTR_DEVICE);
                else erasor.process_scans_retest(bp, raw.data(), off, (int)b0, cfg.updater.query_voxel_size, l2b, cfg.updater.max_range, ERASOR_PTR_DEVICE);
            }
        }
        const ERASOR::DeviceClouds saved = erasor.save_static_map(0.2f);
        const std::string target = cfg.save_path + "/" + cfg.data_name + "_result.pcd";
        codec.write_device(target, saved.d_xyzi, saved.offsets[1]);
        std::cout << sel.size() << " of " << (poses.size() > (size_t)init_idx ? poses.size() - init_idx : 0) << " nodes processed; "
                  << saved.offsets[1] << " points saved to " << target << std::endl;
    } catch (const std::exception& e) {
        std::cerr << e.what() << std::endl;
        return 1;
    }
    return 0;
}
