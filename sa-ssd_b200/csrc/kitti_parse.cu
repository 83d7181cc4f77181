// KITTI label / result text on the device: the reference's get_label_anno (tools/kitti_common.py:560-601) for every
// file of a directory at once, into the flat columns the device evaluator reads (kitti_eval.AnnoBlock):
//
//   sassd_kitti_scan_labels   one thread per file: its readlines() line count, whether its first line has exactly 16
//                             fields (a score column), and whether it must be parsed on the host instead;
//   sassd_kitti_parse_labels  one thread per file writes the bounds of its lines into their row slots, then one thread
//                             per line parses the line.
//
// The device parses a fast grammar only: ASCII text, '\n' line ends, fields separated by single spaces with none
// leading or trailing, every converted field a number [+-]?digits[.digits][(e|E)[+-]?digits] (digits on at least one
// side of the point) with at most 19 significant digits, a significand below 2^53 and a decimal exponent within +-22.
// Such a number is Clinger's fast path: the integer significand and 10^|e| are exact doubles, so one correctly
// rounded multiply or divide gives Python's float() bit for bit.  Every other file is flagged for the host reader, which
// then parses it, or raises, exactly as the reference does.
#include <cmath>
#include <cstdint>

#include "common.cuh"

namespace {

constexpr int kFields = 16;                  // fields the reader converts: name .. rotation_y, then the score
constexpr int kMinFields = 15;               // a line without a score
constexpr int kMaxSig = 19;                  // significant digits of the fast path (w < 10^19 fits in 64 bits)

__constant__ double kPow10[23] = {1e0,  1e1,  1e2,  1e3,  1e4,  1e5,  1e6,  1e7,  1e8,  1e9,  1e10, 1e11,
                                  1e12, 1e13, 1e14, 1e15, 1e16, 1e17, 1e18, 1e19, 1e20, 1e21, 1e22};

__device__ __forceinline__ bool is_digit(uint8_t c) { return c >= '0' && c <= '9'; }

// One field [p, e) as float() reads it, when it is in the fast grammar; false otherwise.
__device__ bool parse_number(const uint8_t* p, const uint8_t* e, double* out) {
    bool neg = false;
    if (p < e && (*p == '+' || *p == '-')) neg = *p++ == '-';
    unsigned long long w = 0;
    int sig = 0, frac = 0, digits = 0;
    for (int part = 0; part < 2; ++part) {   // the integer digits, then the fraction's
        for (; p < e && is_digit(*p); ++p, ++digits) {
            const int d = *p - '0';
            if (part) ++frac;
            if (w == 0 && d == 0) continue; // a leading zero is not significant
            if (++sig > kMaxSig) return false;
            w = w * 10 + d;
        }
        if (part == 0) {
            if (p < e && *p == '.') ++p;
            else break;
        }
    }
    if (digits == 0) return false;
    int ex = 0;
    if (p < e && (*p == 'e' || *p == 'E')) {
        ++p;
        bool eneg = false;
        if (p < e && (*p == '+' || *p == '-')) eneg = *p++ == '-';
        int nd = 0;
        for (; p < e && is_digit(*p); ++p, ++nd)
            if (ex < 100000) ex = ex * 10 + (*p - '0');
        if (nd == 0) return false;
        if (eneg) ex = -ex;
    }
    if (p != e) return false;
    const int e10 = ex - frac;
    if (w >= (1ull << 53) || e10 < -22 || e10 > 22) return false;
    double v = (double)w;
    v = e10 >= 0 ? __dmul_rn(v, kPow10[e10]) : __ddiv_rn(v, kPow10[-e10]);
    *out = neg ? -v : v;                     // the sign last: "-0.00" is -0.0
    return true;
}

// The fields of one line [p, e) ('\n' excluded): the bounds of the first kFields, and the count of all of them.
// False when a field is empty (an empty line, a leading or trailing space, two spaces in a row).
struct Fields {
    int n;
    const uint8_t* b[kFields + 1];           // the starts of the first kFields + 1 fields
};

__device__ bool split_line(const uint8_t* p, const uint8_t* e, Fields& f) {
    f.n = 0;
    const uint8_t* start = p;
    for (;; ++p) {
        if (p == e || *p == ' ') {
            if (p == start) return false;
            if (f.n <= kFields) f.b[f.n] = start;
            ++f.n;
            if (p == e) break;
            start = p + 1;
        }
    }
    return true;
}

__device__ __forceinline__ const uint8_t* field_end(const Fields& f, int i, const uint8_t* line_end) {
    return i + 1 < f.n ? f.b[i + 1] - 1 : line_end;
}

// Every converted value of one line, into out[0 .. 14] (truncated, occluded as int(float()), alpha, bbox[4], h, w, l,
// location[3], rotation_y, score) when out is given; false when the line is outside the fast grammar.
__device__ bool parse_line(const uint8_t* p, const uint8_t* e, bool scored, double* out) {
    Fields f;
    if (!split_line(p, e, f) || f.n < (scored ? kFields : kMinFields)) return false;
    const int last = scored ? kFields : kMinFields;
    for (int i = 1; i < last; ++i) {
        double v;
        if (!parse_number(f.b[i], field_end(f, i, e), &v)) return false;
        if (i == 2) {                        // occluded: int(float(x)), an int64 column
            v = trunc(v) + 0.0;              // int() has no negative zero
            if (fabs(v) >= 9223372036854775808.0) return false;
        }
        if (out) out[i - 1] = v;
    }
    if (out && !scored) out[kMinFields - 1] = 0.0;     // the score
    return true;
}

// One thread per file.  flags: SASSD_KITTI_PARSE_DEFER when the file must be read on the host, SASSD_KITTI_PARSE_SCORE
// when its first line has exactly 16 fields.
__global__ void scan_kernel(const uint8_t* __restrict__ buf, const int64_t* __restrict__ file_off, int nfiles,
                            int32_t* __restrict__ n_lines, int32_t* __restrict__ flags) {
    for (int fi = blockIdx.x * blockDim.x + threadIdx.x; fi < nfiles; fi += gridDim.x * blockDim.x) {
        const uint8_t* p = buf + file_off[fi];
        const uint8_t* end = buf + file_off[fi + 1];
        int lines = 0, flag = 0;
        bool scored = false;
        for (const uint8_t* ls = p; ls < end;) {
            const uint8_t* le = ls;
            bool plain = true;
            for (; le < end && *le != '\n'; ++le)
                if (*le < 0x20 || *le >= 0x7f) plain = false;   // control characters, '\r', tabs and non-ASCII bytes
            if (lines == 0) {
                Fields f;
                scored = split_line(ls, le, f) && f.n == kFields;
            }
            if (!plain || !parse_line(ls, le, scored, nullptr)) {
                flag = SASSD_KITTI_PARSE_DEFER;
                break;
            }
            ++lines;
            ls = le + 1;
        }
        if (scored) flag |= SASSD_KITTI_PARSE_SCORE;
        n_lines[fi] = flag & SASSD_KITTI_PARSE_DEFER ? 0 : lines;
        flags[fi] = flag;
    }
}

// One thread per file that the device parses: line l of file f spans [bounds[2r], bounds[2r + 1]), r = row_off[f] + l.
__global__ void bounds_kernel(const uint8_t* __restrict__ buf, const int64_t* __restrict__ file_off, int nfiles,
                              const int32_t* __restrict__ flags, const int32_t* __restrict__ row_off,
                              int64_t* __restrict__ bounds) {
    for (int fi = blockIdx.x * blockDim.x + threadIdx.x; fi < nfiles; fi += gridDim.x * blockDim.x) {
        if (flags[fi] & SASSD_KITTI_PARSE_DEFER) continue;
        const int64_t end = file_off[fi + 1];
        long long r = row_off[fi];
        for (int64_t ls = file_off[fi]; ls < end; ++r) {
            int64_t le = ls;
            while (le < end && buf[le] != '\n') ++le;
            bounds[2 * r] = ls;
            bounds[2 * r + 1] = le;
            ls = le + 1;
        }
    }
}

__global__ void parse_kernel(const uint8_t* __restrict__ buf, int nfiles, int nrows, const int32_t* __restrict__ flags,
                             const int32_t* __restrict__ row_off, const int64_t* __restrict__ bounds,
                             const char* __restrict__ names, const int32_t* __restrict__ name_off, int nnames,
                             int32_t* __restrict__ name_id, int32_t* __restrict__ dontcare,
                             double* __restrict__ truncated, double* __restrict__ occluded, double* __restrict__ alpha,
                             double* __restrict__ bbox, double* __restrict__ cam, double* __restrict__ score) {
    for (int r = blockIdx.x * blockDim.x + threadIdx.x; r < nrows; r += gridDim.x * blockDim.x) {
        int lo = 0, hi = nfiles;             // the file of row r: row_off[lo] <= r < row_off[lo + 1]
        while (hi - lo > 1) {
            const int mid = (lo + hi) >> 1;
            if (row_off[mid] <= r) lo = mid; else hi = mid;
        }
        if (flags[lo] & SASSD_KITTI_PARSE_DEFER) continue;      // the host fills these rows
        const uint8_t* p = buf + bounds[2 * r];
        const uint8_t* e = buf + bounds[2 * r + 1];
        double v[kFields];
        parse_line(p, e, flags[lo] & SASSD_KITTI_PARSE_SCORE, v);   // the scan accepted every line of the file
        // the name: its lower-cased text against the class-name table, and the exact "DontCare"
        const uint8_t* ne = p;
        while (ne < e && *ne != ' ') ++ne;
        const int len = (int)(ne - p);
        int id = -1;
        for (int j = 0; j < nnames && id < 0; ++j) {
            if (name_off[j + 1] - name_off[j] != len) continue;
            bool same = true;
            for (int i = 0; i < len && same; ++i) {
                uint8_t c = p[i];
                if (c >= 'A' && c <= 'Z') c += 'a' - 'A';
                same = c == (uint8_t)names[name_off[j] + i];
            }
            if (same) id = j;
        }
        const char dc[] = "DontCare";
        bool is_dc = len == 8;
        for (int i = 0; i < 8 && is_dc; ++i) is_dc = p[i] == (uint8_t)dc[i];
        name_id[r] = id;
        dontcare[r] = is_dc;
        truncated[r] = v[0];
        occluded[r] = v[1];
        alpha[r] = v[2];
        for (int i = 0; i < 4; ++i) bbox[4 * (long long)r + i] = v[3 + i];
        double* c = cam + 7 * (long long)r;
        c[0] = v[10]; c[1] = v[11]; c[2] = v[12];                // location
        c[3] = v[9]; c[4] = v[7]; c[5] = v[8];                   // the file's h, w, l as l, h, w
        c[6] = v[13];                                            // rotation_y
        score[r] = v[14];
    }
}

}  // namespace

extern "C" int sassd_kitti_scan_labels(const uint8_t* buf, const int64_t* file_off, int nfiles, int32_t* n_lines,
                                       int32_t* flags, sassd_stream_t stream) {
    if (nfiles < 0 || (nfiles > 0 && (!buf || !file_off || !n_lines || !flags))) return SASSD_ERR_ARG;
    if (nfiles == 0) return SASSD_OK;
    scan_kernel<<<sassd_grid(nfiles, 128), 128, 0, (cudaStream_t)stream>>>(buf, file_off, nfiles, n_lines, flags);
    return sassd_check_launch();
}

extern "C" size_t sassd_kitti_parse_workspace_bytes(int nrows) { return nrows > 0 ? 16 * (size_t)nrows : 0; }

extern "C" int sassd_kitti_parse_labels(const uint8_t* buf, const int64_t* file_off, int nfiles, const int32_t* flags,
                                        const int32_t* row_off, int nrows, const char* names, const int32_t* name_off,
                                        int nnames, int32_t* name_id, int32_t* dontcare, double* truncated,
                                        double* occluded, double* alpha, double* bbox, double* cam, double* score,
                                        void* ws, size_t ws_bytes, sassd_stream_t stream) {
    if (nfiles < 0 || nrows < 0 || nnames < 0 || (nnames > 0 && (!names || !name_off))) return SASSD_ERR_ARG;
    if (nfiles == 0 || nrows == 0) return SASSD_OK;
    if (!buf || !file_off || !flags || !row_off || !name_id || !dontcare || !truncated || !occluded || !alpha ||
        !bbox || !cam || !score || !ws)
        return SASSD_ERR_ARG;
    if (ws_bytes < sassd_kitti_parse_workspace_bytes(nrows)) return SASSD_ERR_WORKSPACE;
    int64_t* bounds = (int64_t*)ws;
    bounds_kernel<<<sassd_grid(nfiles, 128), 128, 0, (cudaStream_t)stream>>>(buf, file_off, nfiles, flags, row_off,
                                                                              bounds);
    parse_kernel<<<sassd_grid(nrows, 128), 128, 0, (cudaStream_t)stream>>>(
        buf, nfiles, nrows, flags, row_off, bounds, names, name_off, nnames, name_id, dontcare, truncated, occluded, alpha,
        bbox, cam, score);
    return sassd_check_launch();
}
