// include/erasor/offline_map_updater.hpp -- ROS-free C++ host mirror of `erasor::OfflineMapUpdater`
// (reference include/erasor/OfflineMapUpdater.h, src/offline_map_updater/src/OfflineMapUpdater.cpp) on top of the
// C ABI in include/erasor_b200.h.  The global map lives on the GPU; `callback_node` takes what an `erasor/node`
// message carries (header.seq, odom, lidar) as plain arguments; `save_static_map` writes the same ASCII PCD the
// reference writes with pcl::io::savePCDFileASCII, which scripts/analysis_runner.py reads, formatted on the device (PcdCodec).
// Everything here goes through the C ABI: no CUDA header or runtime library is needed to use it.
//
// Config: the reference's rosparam tree (config/*.yaml: /erasor/*, /MapUpdater/*, /large_scale/*, /tf/lidar2body,
// /verbose) is read by load_config(); no yaml-cpp is needed for the two-level key: value files the reference ships.
#pragma once
#include <algorithm>
#include <array>
#include <cstdio>
#include <cstring>
#include <fstream>
#include <map>
#include <sstream>
#include <stdexcept>
#include <string>
#include <utility>
#include <vector>

#include "erasor.hpp"

namespace erasor_b200 {

struct Config {
    erasor_params_t         erasor = default_params();
    erasor_updater_params_t updater{};
    std::string data_name = "00", env = "outdoor", initial_map_path = "/", save_path = "/";
    bool verbose = true;
    Config() {
        // defaults of OfflineMapUpdater.cpp:66-83
        updater.query_voxel_size = 0.05; updater.map_voxel_size = 0.05; updater.removal_interval = 2;
        updater.is_large_scale = 0; updater.submap_size = 200.0; updater.max_range = 60.0; updater.version = 3;
        for (int i = 0; i < 7; ++i) updater.lidar2body[i] = 0.0;
        updater.lidar2body[6] = 1.0;
    }
};

namespace detail {
inline std::string trim(const std::string& s) {
    const size_t a = s.find_first_not_of(" \t\r\n"), b = s.find_last_not_of(" \t\r\n");
    return a == std::string::npos ? std::string() : s.substr(a, b - a + 1);
}
inline std::string unquote(std::string v) {
    if (v.size() >= 2 && (v.front() == '"' || v.front() == '\'')) v = v.substr(1, v.size() - 2);
    return v;
}
// "section/key" -> value, for `section:` blocks with indented `key: value` lines; comments (#) stripped
inline std::map<std::string, std::string> read_yaml(const std::string& path) {
    std::ifstream f(path);
    if (!f) throw std::invalid_argument("cannot open config " + path);
    std::map<std::string, std::string> kv;
    std::string line, section;
    while (std::getline(f, line)) {
        const size_t hash = line.find('#');
        if (hash != std::string::npos) line = line.substr(0, hash);
        if (trim(line).empty()) continue;
        const bool indented = line[0] == ' ' || line[0] == '\t';
        const size_t colon = line.find(':');
        if (colon == std::string::npos) continue;
        const std::string key = trim(line.substr(0, colon)), val = trim(line.substr(colon + 1));
        if (!indented) { section = val.empty() ? key : std::string(); if (!val.empty()) kv[key] = val; }
        else kv[section + "/" + key] = val;
    }
    return kv;
}
}  // namespace detail

inline Config load_config(const std::string& yaml_path) {
    const auto kv = detail::read_yaml(yaml_path);
    Config c;
    auto num = [&](const char* k, double& dst) { auto it = kv.find(k); if (it != kv.end()) dst = std::stod(it->second); };
    auto inum = [&](const char* k, int& dst) { auto it = kv.find(k); if (it != kv.end()) dst = (int)std::stod(it->second); };
    auto str = [&](const char* k, std::string& dst) { auto it = kv.find(k); if (it != kv.end()) dst = detail::unquote(it->second); };
    erasor_params_t& e = c.erasor;
    num("erasor/max_range", e.max_range); inum("erasor/num_rings", e.num_rings); inum("erasor/num_sectors", e.num_sectors);
    num("erasor/max_h", e.max_h); num("erasor/min_h", e.min_h); num("erasor/th_bin_max_h", e.th_bin_max_h);
    num("erasor/scan_ratio_threshold", e.scan_ratio_threshold); inum("erasor/num_lowest_pts", e.num_lowest_pts);
    inum("erasor/minimum_num_pts", e.minimum_num_pts); num("erasor/rejection_ratio", e.rejection_ratio);
    num("erasor/gf_dist_thr", e.gf_dist_thr); inum("erasor/gf_iter", e.gf_iter); inum("erasor/gf_num_lpr", e.gf_num_lpr);
    num("erasor/gf_th_seeds_height", e.gf_th_seeds_height); num("erasor/map_voxel_size", e.map_voxel_size);
    inum("erasor/version", e.version);
    erasor_updater_params_t& u = c.updater;
    num("MapUpdater/query_voxel_size", u.query_voxel_size); num("MapUpdater/map_voxel_size", u.map_voxel_size);
    inum("MapUpdater/removal_interval", u.removal_interval);
    str("MapUpdater/data_name", c.data_name); str("MapUpdater/env", c.env);
    str("MapUpdater/initial_map_path", c.initial_map_path); str("MapUpdater/save_path", c.save_path);
    { auto it = kv.find("large_scale/is_large_scale"); if (it != kv.end()) u.is_large_scale = (it->second == "true" || it->second == "True" || it->second == "1"); }
    num("large_scale/submap_size", u.submap_size);
    u.max_range = 60.0; num("erasor/max_range", u.max_range);            // the updater's own default differs (App. B-8)
    u.version = e.version;
    { auto it = kv.find("verbose"); if (it != kv.end()) c.verbose = (it->second != "false" && it->second != "False" && it->second != "0"); }
    auto it = kv.find("tf/lidar2body");
    if (it != kv.end()) {
        std::string v = it->second;
        for (char& ch : v) if (ch == '[' || ch == ']' || ch == ',') ch = ' ';
        std::istringstream ss(v);
        std::vector<double> vals; double d;
        while (ss >> d) vals.push_back(d);
        if (vals.size() == 7) for (int i = 0; i < 7; ++i) u.lidar2body[i] = vals[i];
    }
    return c;
}

// PCD readers / writer for the file layouts the reference uses (ASCII and binary, FIELDS containing x y z intensity).  load_pcd's
// binary branch ignores COUNT and copies intensity as four raw bytes whatever its TYPE; PcdCodec::load follows PCL's rules instead
// (DESIGN.md section 12.1 records the divergence).
inline PointCloud load_pcd(const std::string& path) {
    std::ifstream f(path, std::ios::binary);
    if (!f) throw std::invalid_argument("Maybe intiial map path is not correct!");      // OfflineMapUpdater.cpp:125 (sic)
    std::vector<std::string> fields; std::vector<int> sizes; size_t n = 0; std::string mode, line;
    while (std::getline(f, line)) {
        std::istringstream ss(line); std::string tag; ss >> tag;
        if (tag == "FIELDS") { std::string s; while (ss >> s) fields.push_back(s); }
        else if (tag == "SIZE") { int s; while (ss >> s) sizes.push_back(s); }
        else if (tag == "POINTS") ss >> n;
        else if (tag == "DATA") { ss >> mode; break; }
    }
    int ix = -1, iy = -1, iz = -1, ii = -1;
    for (size_t k = 0; k < fields.size(); ++k) {
        if (fields[k] == "x") ix = (int)k; else if (fields[k] == "y") iy = (int)k; else if (fields[k] == "z") iz = (int)k;
        else if (fields[k] == "intensity") ii = (int)k;
    }
    if (ix < 0 || iy < 0 || iz < 0) throw std::invalid_argument("PCD without x y z fields: " + path);
    PointCloud c(n);
    if (mode == "ascii") {
        std::vector<double> row(fields.size());
        for (size_t i = 0; i < n; ++i) {
            for (auto& v : row) f >> v;
            c[i] = {(float)row[ix], (float)row[iy], (float)row[iz], ii >= 0 ? (float)row[ii] : 0.0f};
        }
    } else if (mode == "binary") {
        size_t stride = 0; std::vector<size_t> off(fields.size());
        for (size_t k = 0; k < fields.size(); ++k) { off[k] = stride; stride += (k < sizes.size() ? sizes[k] : 4); }
        std::vector<char> buf(stride);
        for (size_t i = 0; i < n; ++i) {
            f.read(buf.data(), stride);
            auto get = [&](int k) { float v; std::memcpy(&v, buf.data() + off[k], 4); return v; };
            c[i] = {get(ix), get(iy), get(iz), ii >= 0 ? get(ii) : 0.0f};
        }
    } else {
        throw std::invalid_argument("unsupported PCD DATA mode '" + mode + "' in " + path);
    }
    return c;
}
inline void save_pcd_ascii(const std::string& path, const PointCloud& c) {
    std::ofstream f(path);
    if (!f) throw std::runtime_error("cannot write " + path);
    f << "# .PCD v0.7 - Point Cloud Data file format\nVERSION 0.7\nFIELDS x y z intensity\nSIZE 4 4 4 4\nTYPE F F F F\nCOUNT 1 1 1 1\n"
      << "WIDTH " << c.size() << "\nHEIGHT 1\nVIEWPOINT 0 0 0 1 0 0 0\nPOINTS " << c.size() << "\nDATA ascii\n";
    f.precision(8);
    for (const auto& p : c) f << p.x << ' ' << p.y << ' ' << p.z << ' ' << p.intensity << '\n';
}

// PCD files through the device codec (erasor_pcd_*).  read / read_device parse ASCII files and give what load_pcd gives bit for bit
// (intensity 0 when the file has none); binary files are UnsupportedPcd there.  load / load_device read every DATA mode (ascii,
// binary, binary_compressed) with PCL's field rules (DESIGN.md section 12.1).  The writer gives the bytes save_pcd_ascii writes
// (NaN spelled "nan"), or a binary or binary_compressed file (DESIGN.md section 12.3).
struct UnsupportedPcd : std::runtime_error { using std::runtime_error::runtime_error; };

class PcdCodec {
public:
    explicit PcdCodec(int device = 0) {
        if (erasor_pcd_create(device, &p_) != ERASOR_OK) throw std::runtime_error(std::string("PcdCodec: ") + erasor_pcd_last_error(nullptr));
    }
    ~PcdCodec() { erasor_pcd_destroy(p_); }
    PcdCodec(const PcdCodec&) = delete;
    PcdCodec& operator=(const PcdCodec&) = delete;

    // The file at path into device memory.  device_buffer(n) must return a 16-byte aligned device pointer with room for n points
    // (the caller owns the memory); returns the points parsed.  Synchronous: the cloud is complete on return.
    template <class DeviceBuffer>
    size_t read_device(const std::string& path, DeviceBuffer&& device_buffer) {
        slurp(path);
        size_t n = 0;
        check(erasor_pcd_parse_ascii(p_, text_.data(), text_.size(), ERASOR_PTR_HOST, nullptr, 0, ERASOR_PTR_DEVICE, &n, nullptr), path);
        float* out = device_buffer(n);
        check(erasor_pcd_parse_ascii(p_, text_.data(), text_.size(), ERASOR_PTR_HOST, out, n, ERASOR_PTR_DEVICE, &n, nullptr), path);
        return n;
    }
    PointCloud read(const std::string& path) {
        slurp(path);
        size_t n = 0;
        check(erasor_pcd_parse_ascii(p_, text_.data(), text_.size(), ERASOR_PTR_HOST, nullptr, 0, ERASOR_PTR_HOST, &n, nullptr), path);
        PointCloud c(n);
        check(erasor_pcd_parse_ascii(p_, text_.data(), text_.size(), ERASOR_PTR_HOST, reinterpret_cast<float*>(c.data()), n, ERASOR_PTR_HOST, &n, nullptr), path);
        c.resize(n);
        return c;
    }
    // erasor_pcd_load: the file at path, in any DATA mode, into device memory (device_buffer as for read_device) or a host cloud
    template <class DeviceBuffer>
    size_t load_device(const std::string& path, DeviceBuffer&& device_buffer) {
        slurp(path);
        size_t n = 0;
        check(erasor_pcd_load(p_, text_.data(), text_.size(), ERASOR_PTR_HOST, nullptr, 0, ERASOR_PTR_DEVICE, &n, nullptr), path);
        float* out = device_buffer(n);
        check(erasor_pcd_load(p_, text_.data(), text_.size(), ERASOR_PTR_HOST, out, n, ERASOR_PTR_DEVICE, &n, nullptr), path);
        return n;
    }
    PointCloud load(const std::string& path) {
        slurp(path);
        size_t n = 0;
        check(erasor_pcd_load(p_, text_.data(), text_.size(), ERASOR_PTR_HOST, nullptr, 0, ERASOR_PTR_HOST, &n, nullptr), path);
        PointCloud c(n);
        check(erasor_pcd_load(p_, text_.data(), text_.size(), ERASOR_PTR_HOST, reinterpret_cast<float*>(c.data()), n, ERASOR_PTR_HOST, &n, nullptr), path);
        c.resize(n);
        return c;
    }
    // data_mode: ERASOR_PCD_ASCII (save_pcd_ascii's bytes), ERASOR_PCD_BINARY or ERASOR_PCD_BINARY_COMPRESSED (erasor_pcd_format)
    void write(const std::string& path, const PointCloud& c, int data_mode = ERASOR_PCD_ASCII) {
        write_from(path, reinterpret_cast<const float*>(c.data()), c.size(), ERASOR_PTR_HOST, data_mode);
    }
    // the same file from n points in device memory (e.g. ERASOR::save_static_map's cloud)
    void write_device(const std::string& path, const float* d_xyzi, size_t n, int data_mode = ERASOR_PCD_ASCII) {
        write_from(path, d_xyzi, n, ERASOR_PTR_DEVICE, data_mode);
    }

private:
    void write_from(const std::string& path, const float* src, size_t n, int in_kind, int data_mode) {
        size_t len = 0;
        check(erasor_pcd_format(p_, src, n, in_kind, data_mode, nullptr, 0, ERASOR_PTR_HOST, &len, nullptr), path);
        text_.resize(len);
        check(erasor_pcd_format(p_, src, n, in_kind, data_mode, text_.data(), len, ERASOR_PTR_HOST, &len, nullptr), path);
        std::ofstream f(path, std::ios::binary);
        if (!f || !f.write(text_.data(), (std::streamsize)len)) throw std::runtime_error("cannot write " + path);
    }
    void slurp(const std::string& path) {
        std::ifstream f(path, std::ios::binary | std::ios::ate);
        if (!f) throw std::invalid_argument("cannot open " + path);
        text_.resize((size_t)f.tellg());
        f.seekg(0);
        if (!text_.empty() && !f.read(text_.data(), (std::streamsize)text_.size())) throw std::runtime_error("cannot read " + path);
    }
    void check(int rc, const std::string& path) const {
        if (rc == ERASOR_OK) return;
        const std::string msg = path + ": " + erasor_pcd_last_error(p_);
        if (rc == ERASOR_E_UNSUPPORTED) throw UnsupportedPcd(msg);
        if (rc == ERASOR_E_INVALID) throw std::invalid_argument(msg);
        throw std::runtime_error(msg);
    }
    erasor_pcd_t p_ = nullptr;
    std::vector<char> text_;
};

// A ROS bag of erasor/node messages (the reference's <seq>_..._node.bag, DESIGN.md section 12.2): indexed on the host when
// constructed, clouds decoded on the device (erasor_bag_*).  The nodes are the messages on `topic` as the reference's subscribers
// receive them: the first one is dropped unless keep_first.
struct BagNode {
    uint32_t seq;                    // header.seq
    std::array<double, 7> odom;      // x y z qx qy qz qw, as stored
};

class NodeBag {
public:
    explicit NodeBag(const std::string& path, const std::string& topic = "/node/combined/optimized", bool keep_first = false, int device = 0)
        : path_(path) {
        if (erasor_pcd_create(device, &p_) != ERASOR_OK) throw std::runtime_error(std::string("NodeBag: ") + erasor_pcd_last_error(nullptr));
        std::ifstream f(path, std::ios::binary | std::ios::ate);
        if (!f) { erasor_pcd_destroy(p_); throw std::invalid_argument("cannot open " + path); }
        file_.resize((size_t)f.tellg());
        f.seekg(0);
        if (!file_.empty() && !f.read(file_.data(), (std::streamsize)file_.size())) { erasor_pcd_destroy(p_); throw std::runtime_error("cannot read " + path); }
        size_t n = 0;
        int rc = erasor_bag_index(p_, file_.data(), file_.size(), topic.c_str(), keep_first ? 1 : 0, &n, &info_);
        std::vector<uint32_t> seq(n);
        std::vector<double> odom(7 * n);
        if (rc == ERASOR_OK) rc = erasor_bag_nodes(p_, 0, n, seq.data(), nullptr, odom.data(), nullptr);
        if (rc != ERASOR_OK) {
            const std::string msg = path + ": " + erasor_pcd_last_error(p_);
            erasor_pcd_destroy(p_);
            if (rc == ERASOR_E_UNSUPPORTED) throw UnsupportedPcd(msg);
            if (rc == ERASOR_E_INVALID) throw std::invalid_argument(msg);
            throw std::runtime_error(msg);
        }
        nodes_.resize(n);
        for (size_t i = 0; i < n; ++i) {
            nodes_[i].seq = seq[i];
            std::copy(odom.begin() + 7 * i, odom.begin() + 7 * i + 7, nodes_[i].odom.begin());
        }
    }
    ~NodeBag() { erasor_pcd_destroy(p_); }
    NodeBag(const NodeBag&) = delete;
    NodeBag& operator=(const NodeBag&) = delete;

    size_t size() const { return nodes_.size(); }
    const BagNode& node(size_t i) const { return nodes_.at(i); }
    const erasor_bag_info_t& info() const { return info_; }
    // the bag's lz4 chunks: how many were uploaded and decoded, bytes, blocks, checksums (erasor_bag_lz4_stats)
    erasor_bag_lz4_stats_t lz4_stats() const {
        erasor_bag_lz4_stats_t s{};
        check(erasor_bag_lz4_stats(p_, &s));
        return s;
    }
    // the bag's bz2 chunks: how many were uploaded and decoded, bytes, blocks and candidates, scratch, stage times (erasor_bag_bz2_stats)
    erasor_bag_bz2_stats_t bz2_stats() const {
        erasor_bag_bz2_stats_t s{};
        check(erasor_bag_bz2_stats(p_, &s));
        return s;
    }
    // The clouds of nodes [first, first + count) -- or of the listed nodes -- back to back in device memory, from one gather
    // launch.  device_buffer(n) must return a 16-byte aligned device pointer with room for n points (the caller owns the memory).
    // Returns the count + 1 offsets.  Synchronous: the clouds are complete on return.
    template <class DeviceBuffer>
    std::vector<uint64_t> load_device(size_t first, size_t count, DeviceBuffer&& device_buffer) {
        std::vector<uint64_t> list(count);
        for (size_t k = 0; k < count; ++k) list[k] = first + k;
        return load_device(list, std::forward<DeviceBuffer>(device_buffer));
    }
    template <class DeviceBuffer>
    std::vector<uint64_t> load_device(const std::vector<uint64_t>& nodes, DeviceBuffer&& device_buffer) {
        std::vector<uint64_t> off(nodes.size() + 1, 0);
        check(erasor_bag_load_list(p_, nodes.data(), nodes.size(), nullptr, 0, ERASOR_PTR_DEVICE, off.data()));
        float* out = device_buffer((size_t)off.back());
        check(erasor_bag_load_list(p_, nodes.data(), nodes.size(), out, (size_t)off.back(), ERASOR_PTR_DEVICE, off.data()));
        return off;
    }

private:
    void check(int rc) const {
        if (rc == ERASOR_OK) return;
        const std::string msg = path_ + ": " + erasor_pcd_last_error(p_);
        if (rc == ERASOR_E_INVALID) throw std::invalid_argument(msg);
        throw std::runtime_error(msg);
    }
    std::string path_;
    erasor_pcd_t p_ = nullptr;
    std::vector<char> file_;
    erasor_bag_info_t info_{};
    std::vector<BagNode> nodes_;
};

inline bool is_bag_path(const std::string& path) { return path.size() > 4 && path.compare(path.size() - 4, 4, ".bag") == 0; }

class OfflineMapUpdater {
public:
    // replaces OfflineMapUpdater::OfflineMapUpdater(): set_params + load_global_map + new ERASOR (OfflineMapUpdater.cpp:5-32)
    OfflineMapUpdater(const Config& cfg, const PointCloud& initial_map, int device = 0) : cfg_(cfg), device_(device) {
        if (cfg.env != "outdoor") throw std::invalid_argument("This `indoor` mode is not perfect!");   // :149
        const int rc = erasor_updater_create(&cfg_.updater, &cfg_.erasor, reinterpret_cast<const float*>(initial_map.data()),
                                             initial_map.size(), device, &u_);
        if (rc == ERASOR_E_INVALID) throw std::invalid_argument(std::string("OfflineMapUpdater: ") + erasor_updater_last_error(nullptr));
        if (rc != ERASOR_OK) throw std::runtime_error(std::string("OfflineMapUpdater: ") + erasor_updater_last_error(nullptr));
    }
    explicit OfflineMapUpdater(const Config& cfg, int device = 0) : OfflineMapUpdater(cfg, load_pcd(cfg.initial_map_path), device) {}
    ~OfflineMapUpdater() { erasor_updater_destroy(u_); }
    OfflineMapUpdater(const OfflineMapUpdater&) = delete;
    OfflineMapUpdater& operator=(const OfflineMapUpdater&) = delete;

    // replaces callback_node(const erasor::node::ConstPtr&) (:203-330): odom = {x y z qx qy qz qw} body -> origin,
    // lidar in the lidar frame.  Returns true when the node was processed, false for "PASS!".
    bool callback_node(int seq, const double odom[7], const PointCloud& lidar) {
        ++calls_;
        int processed = 0;
        check(erasor_updater_process_node(u_, seq, odom, reinterpret_cast<const float*>(lidar.data()), lidar.size(), ERASOR_PTR_HOST, &processed));
        if (cfg_.verbose) std::printf(processed ? "\033[01;32m%dth frame\033[0m is comming\n" : "\033[1;32m PASS! \033[0m\n", seq);
        return processed != 0;
    }
    // Look-ahead (no counterpart in the reference, which receives its nodes one ROS message at a time): hand in the scan of a COMING
    // callback_node call so that its upload and voxelisation (:237-241) run under the current node's path.  `lidar` must stay
    // alive and unchanged until that call; results are identical with and without.
    void prefetch(const PointCloud& lidar) { check(erasor_updater_prefetch_scan(u_, reinterpret_cast<const float*>(lidar.data()), lidar.size(), ERASOR_PTR_HOST)); }
    // the same two calls with a scan of n points already in device memory (e.g. parsed there by PcdCodec::read_device); the scan
    // must be complete before prefetch_device, and stay unchanged until its callback_node_device call
    bool callback_node_device(int seq, const double odom[7], const float* lidar_xyzi, size_t n) {
        ++calls_;
        int processed = 0;
        check(erasor_updater_process_node(u_, seq, odom, lidar_xyzi, n, ERASOR_PTR_DEVICE, &processed));
        if (cfg_.verbose) std::printf(processed ? "\033[01;32m%dth frame\033[0m is comming\n" : "\033[1;32m PASS! \033[0m\n", seq);
        return processed != 0;
    }
    void prefetch_device(const float* lidar_xyzi, size_t n) { check(erasor_updater_prefetch_scan(u_, lidar_xyzi, n, ERASOR_PTR_DEVICE)); }
    // will the k-th callback_node call from now (k = 1: the next one) process its node, or "PASS!" (removal_interval, :328)?
    bool processes_call(int k) const { return (calls_ + k) % cfg_.updater.removal_interval == 0; }
    // replaces save_static_map(float voxel_size) (:174-196)
    void save_static_map(float voxel_size) {
        PointCloud map_to_be_saved = static_map(voxel_size);
        const std::string target = cfg_.save_path + "/" + cfg_.data_name + "_result.pcd";
        std::printf("\033[1;32mTARGET: %s\033[0m\nVoxelization operated with %g voxel size\n", target.c_str(), voxel_size);
        PcdCodec(device_).write(target, map_to_be_saved);            // the bytes save_pcd_ascii writes, formatted on the device
        std::printf("\033[1;32mComplete to save the final static map\033[0m\n");
    }
    PointCloud static_map(float voxel_size) {
        size_t n = 0;
        check(erasor_updater_save_static_map(u_, voxel_size, nullptr, 0, &n));
        PointCloud out(n);
        if (n) check(erasor_updater_save_static_map(u_, voxel_size, reinterpret_cast<float*>(out.data()), n, &n));
        return out;
    }
    PointCloud map_arranged() {
        size_t n = 0;
        check(erasor_updater_get_cloud(u_, 0, nullptr, 0, &n, ERASOR_PTR_HOST));
        PointCloud out(n);
        if (n) check(erasor_updater_get_cloud(u_, 0, reinterpret_cast<float*>(out.data()), n, &n, ERASOR_PTR_HOST));
        return out;
    }
    erasor_updater_t handle() const { return u_; }

private:
    void check(int rc) const {
        if (rc == ERASOR_OK) return;
        const std::string msg = std::string("OfflineMapUpdater: ") + erasor_updater_last_error(u_);
        if (rc == ERASOR_E_INVALID) throw std::invalid_argument(msg);
        throw std::runtime_error(msg);
    }
    Config cfg_;
    erasor_updater_t u_ = nullptr;
    int device_ = 0;
    long long calls_ = 0;          // callback_node calls so far (the updater's stack_count, :206)
};

}  // namespace erasor_b200

// The reference declares `namespace erasor { class OfflineMapUpdater; }` (OfflineMapUpdater.h:8).  With
// ERASOR_B200_GLOBAL_NAMES defined, the same qualified name resolves to this class, so that main()-level code written
// against the reference (`erasor::OfflineMapUpdater updater;`) only changes its constructor argument.
#ifdef ERASOR_B200_GLOBAL_NAMES
namespace erasor { using OfflineMapUpdater = erasor_b200::OfflineMapUpdater; }
#endif
