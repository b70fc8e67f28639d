// host_selftest.cpp -- compiles binning.h and pcd_codec.h for the HOST so that the CPU test-suite (-m "not gpu")
// can check the exact-threshold bin arithmetic against the oracle, and the ASCII PCD codec's per-token arithmetic against
// numpy and Python, without a GPU.
// This library is loaded by tests only; the product API (erasor_capi.cu) has no host compute path.
#include <cstdint>
#include <cstring>
#include <string>

#include "binning_tables.h"
#include "pcd_codec.h"
#include "pose_math.h"

extern "C" {

// bins[i] = bin id or -1; stats = {negzero, ambiguous, slow}; qerr_max = max |q_float - q_double| over binned points
int erasor_hostcheck_bin_points(const erasor_params_t* p, const float* xyzi, size_t n, int32_t* bins,
                                uint64_t* stats3, double* qerr_max, double* eps_q) {
    erasor::HostBinTables T;
    std::string err;
    if (erasor::build_bin_tables(*p, T, err) != 0) return -1;
    const erasor::BinTablesView v = T.host_view();
    erasor::BinFenceCounters fc{0, 0, 0};
    uint64_t s0 = 0, s1 = 0, s2 = 0;
    double qe = 0.0;
    for (size_t i = 0; i < n; ++i) {
        fc = erasor::BinFenceCounters{0, 0, 0};
        const float x = xyzi[4 * i], y = xyzi[4 * i + 1], z = xyzi[4 * i + 2];
        bins[i] = erasor::bin_of_point(v, v.ring_thr, x, y, z, &fc);
        s0 += fc.negzero; s1 += fc.ambiguous; s2 += fc.slow;
        if (bins[i] >= 0 && y != 0.0f) {
            // replicate the float guess and compare with the double-precision coordinate
            const float ax = std::fabs(x), ay = std::fabs(y);
            const float mx = std::fmax(ax, ay), mn = std::fmin(ax, ay);
            float a = erasor::atan_unit(mn / mx);
            if (ay > ax) a = 1.57079637f - a;
            if (x < 0.0f) a = 3.14159274f - a;
            if (y < 0.0f) a = 6.28318548f - a;
            const float  q  = a * v.inv_ss;
            const double th = (y >= 0) ? std::atan2((double)y, (double)x) : 2 * 3.1415926535 + std::atan2((double)y, (double)x);
            const double e  = std::fabs((double)q - th / T.sector_size);
            if (e > qe) qe = e;
        }
    }
    stats3[0] = s0; stats3[1] = s1; stats3[2] = s2;
    *qerr_max = qe;
    *eps_q = T.eps_q;
    return 0;
}

// expose the tables for inspection: ring thresholds (R+1 doubles), s_max, z window
int erasor_hostcheck_tables(const erasor_params_t* p, double* ring_thr, double* s_max, float* z_lo, float* z_hi, int* sec_of_pi) {
    erasor::HostBinTables T;
    std::string err;
    if (erasor::build_bin_tables(*p, T, err) != 0) return -1;
    std::memcpy(ring_thr, T.ring_thr.data(), sizeof(double) * (T.R + 1));
    *s_max = T.s_max; *z_lo = T.z_lo; *z_hi = T.z_hi; *sec_of_pi = T.sec_of_pi;
    return 0;
}

// what erasor_process_nodes hands the device for one node (pose_math.h): criterion point, squared radius, origin -> body rows and the
// float guard band of the radius pre-test
int erasor_hostcheck_node_pose(const double* odom7, double voi_max_range, double* px_py_limit, float* T12, float* guards4) {
    erasor::NodePose np;
    erasor::node_pose_of(odom7, voi_max_range, np);
    px_py_limit[0] = np.px; px_py_limit[1] = np.py; px_py_limit[2] = np.limit;
    for (int i = 0; i < 12; ++i) T12[i] = np.T[i];
    guards4[0] = np.pxf; guards4[1] = np.pyf; guards4[2] = np.lim_lo; guards4[3] = np.lim_hi;
    return 0;
}

// the float guard bands of the device's fast path (binning_tables.cpp): {up_k, dn_k} per ring threshold and around s_max
int erasor_hostcheck_guards(const erasor_params_t* p, float* ring_guard, float* smax_lo_hi) {
    erasor::HostBinTables T;
    std::string err;
    if (erasor::build_bin_tables(*p, T, err) != 0) return -1;
    std::memcpy(ring_guard, T.ring_guard.data(), sizeof(float) * T.ring_guard.size());
    smax_lo_hi[0] = T.smax_lo; smax_lo_hi[1] = T.smax_hi;
    return 0;
}

// pcd_codec.h's parse on n tokens, token k = text[offs[k] .. offs[k + 1]): bits[k] = the float's bit pattern (0 when invalid),
// kind[k] = 0 fast path, 1 big-integer path, 2 invalid.  want_value = 0 runs the check alone, as the kernel does for a column it
// does not keep (kind 0 or 2, bits 0).
int erasor_hostcheck_pcd_parse(const uint8_t* text, const uint64_t* offs, size_t n, int want_value, uint32_t* bits, int32_t* kind) {
    pcd::Big D, A, B;
    for (size_t k = 0; k < n; ++k) {
        const uint8_t* s = text + offs[k];
        const uint64_t len = offs[k + 1] - offs[k];
        const pcd::TokenScan r = pcd::scan_token(s, len, want_value != 0);
        kind[k] = r.kind;
        float f = 0.0f;
        if (r.kind == pcd::TOK_OK && want_value) f = (float)r.value;
        else if (r.kind == pcd::TOK_SLOW) {
            const double v = pcd::parse_slow_abs(s, len, D, A, B);
            f = (float)(r.neg ? -v : v);
        }
        bits[k] = pcd::float_to_bits(f);
    }
    return 0;
}

// pcd_codec.h's "%.8g" on n floats: value k's text at out[16 k ..], its length in lens[k]
int erasor_hostcheck_pcd_format(const float* vals, size_t n, char* out, int32_t* lens) {
    for (size_t k = 0; k < n; ++k) lens[k] = pcd::format_g8(vals[k], out + 16 * k);
    return 0;
}
}
