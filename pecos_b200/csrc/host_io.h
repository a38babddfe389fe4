// Host-side readers for the on-disk formats the two hot paths consume.
//
//   * JsonValue / json_parse      - param.json / config.json
//                                   (reference parses these with nlohmann json:
//                                    pecos/core/xmc/inference.hpp:59-177, pecos/core/ann/hnsw.hpp:470-488)
//   * NpzFile                     - uncompressed scipy .npz (zip "stored" members holding .npy arrays)
//                                   (format consumed by pecos/core/utils/scipy_loader.hpp:207-341)
//   * MmapStoreReader             - PECOS "*.mmap_store" container
//                                   (format defined by pecos/core/utils/mmap_util.hpp:54-184, :190-283)
//
// Everything here is plain host C++17: no CUDA, no torch.  Errors are reported by throwing
// std::runtime_error; the C-ABI layer (c_api.cu) turns them into a message on stderr + abort(),
// which mirrors the reference (C++ exceptions escaping extern "C" => std::terminate).
#pragma once

#include <atomic>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <map>
#include <memory>
#include <stdexcept>
#include <string>
#include <thread>
#include <vector>

#include <fcntl.h>
#include <sys/mman.h>
#include <sys/stat.h>
#include <unistd.h>

namespace pb200 {

// Host view of a caller's matrix (queries, codes or a selected-outputs pattern): CSR (row_ptr/col_idx/val, absolute
// offsets) or row-major dense (dense).  An empty HostMatrix stands for "not given".
struct HostMatrix {
    const uint64_t* row_ptr = nullptr;
    const uint32_t* col_idx = nullptr;
    const float* val = nullptr;
    const float* dense = nullptr;
    uint32_t rows = 0;
    uint32_t cols = 0;

    // rows [r0, r1) (CSR: the offsets stay absolute into col_idx / val)
    HostMatrix row_block(uint32_t r0, uint32_t r1) const {
        HostMatrix b = *this;
        if (row_ptr) b.row_ptr = row_ptr + r0;
        else b.dense = dense + static_cast<uint64_t>(r0) * cols;
        b.rows = r1 - r0;
        return b;
    }
};

// ----------------------------------------------------------------------------------------------
// Read-only memory mapped file
// ----------------------------------------------------------------------------------------------
class MappedFile {
public:
    MappedFile() = default;
    MappedFile(const MappedFile&) = delete;
    MappedFile& operator=(const MappedFile&) = delete;
    ~MappedFile() { close_(); }

    void open(const std::string& path, bool populate) {
        close_();
        int fd = ::open(path.c_str(), O_RDONLY);
        if (fd < 0) throw std::runtime_error("cannot open " + path);
        struct stat st;
        if (fstat(fd, &st) != 0) { ::close(fd); throw std::runtime_error("cannot stat " + path); }
        size_ = static_cast<uint64_t>(st.st_size);
        if (size_ == 0) { ::close(fd); throw std::runtime_error("empty file " + path); }
        int flags = MAP_PRIVATE;
        if (populate) flags |= MAP_POPULATE;
        void* p = mmap(nullptr, size_, PROT_READ, flags, fd, 0);
        ::close(fd);
        if (p == MAP_FAILED) throw std::runtime_error("mmap failed for " + path);
        ptr_ = static_cast<const uint8_t*>(p);
        path_ = path;
    }
    const uint8_t* data() const { return ptr_; }
    uint64_t size() const { return size_; }
    const std::string& path() const { return path_; }
    bool is_open() const { return ptr_ != nullptr; }

private:
    void close_() {
        if (ptr_) munmap(const_cast<uint8_t*>(ptr_), size_);
        ptr_ = nullptr;
        size_ = 0;
    }
    const uint8_t* ptr_ = nullptr;
    uint64_t size_ = 0;
    std::string path_;
};

inline bool file_exists(const std::string& path) { return access(path.c_str(), F_OK) == 0; }

inline std::string read_text_file(const std::string& path) {
    FILE* fp = fopen(path.c_str(), "rb");
    if (!fp) throw std::runtime_error("could not open " + path);
    std::string s;
    char buf[4096];
    size_t n;
    while ((n = fread(buf, 1, sizeof(buf), fp)) > 0) s.append(buf, n);
    fclose(fp);
    return s;
}

// ----------------------------------------------------------------------------------------------
// Minimal JSON (objects, arrays, strings, numbers, true/false/null)
// ----------------------------------------------------------------------------------------------
struct JsonValue {
    enum Kind { Null, Bool, Number, String, Array, Object } kind = Null;
    bool b = false;
    double num = 0.0;
    std::string str;
    std::vector<JsonValue> arr;
    std::vector<std::pair<std::string, JsonValue>> obj;

    const JsonValue* find(const std::string& key) const {
        if (kind != Object) return nullptr;
        for (auto& kv : obj) if (kv.first == key) return &kv.second;
        return nullptr;
    }
    bool contains(const std::string& key) const { return find(key) != nullptr; }
    const JsonValue& at(const std::string& key) const {
        const JsonValue* v = find(key);
        if (!v) throw std::runtime_error("json: missing key '" + key + "'");
        return *v;
    }
    std::string as_string() const {
        if (kind != String) throw std::runtime_error("json: value is not a string");
        return str;
    }
    double as_number() const {
        if (kind == Number) return num;
        if (kind == Bool) return b ? 1.0 : 0.0;
        throw std::runtime_error("json: value is not a number");
    }
    bool as_bool() const {
        if (kind == Bool) return b;
        if (kind == Number) return num != 0.0;
        throw std::runtime_error("json: value is not a bool");
    }
};

class JsonParser {
public:
    explicit JsonParser(const std::string& text) : s_(text) {}
    JsonValue parse() {
        JsonValue v = value_();
        ws_();
        if (p_ != s_.size()) fail_("trailing characters");
        return v;
    }

private:
    const std::string& s_;
    size_t p_ = 0;

    [[noreturn]] void fail_(const char* what) const {
        throw std::runtime_error(std::string("json parse error: ") + what + " at offset " + std::to_string(p_));
    }
    void ws_() { while (p_ < s_.size() && (s_[p_] == ' ' || s_[p_] == '\n' || s_[p_] == '\t' || s_[p_] == '\r')) ++p_; }
    bool lit_(const char* w) {
        size_t n = strlen(w);
        if (s_.compare(p_, n, w) == 0) { p_ += n; return true; }
        return false;
    }
    JsonValue value_() {
        ws_();
        if (p_ >= s_.size()) fail_("unexpected end");
        char c = s_[p_];
        JsonValue v;
        if (c == '{') {
            v.kind = JsonValue::Object;
            ++p_; ws_();
            if (p_ < s_.size() && s_[p_] == '}') { ++p_; return v; }
            for (;;) {
                ws_();
                if (p_ >= s_.size() || s_[p_] != '"') fail_("expected object key");
                std::string k = string_();
                ws_();
                if (p_ >= s_.size() || s_[p_] != ':') fail_("expected ':'");
                ++p_;
                JsonValue item = value_();
                v.obj.emplace_back(std::move(k), std::move(item));
                ws_();
                if (p_ < s_.size() && s_[p_] == ',') { ++p_; continue; }
                if (p_ < s_.size() && s_[p_] == '}') { ++p_; break; }
                fail_("expected ',' or '}'");
            }
        } else if (c == '[') {
            v.kind = JsonValue::Array;
            ++p_; ws_();
            if (p_ < s_.size() && s_[p_] == ']') { ++p_; return v; }
            for (;;) {
                v.arr.push_back(value_());
                ws_();
                if (p_ < s_.size() && s_[p_] == ',') { ++p_; continue; }
                if (p_ < s_.size() && s_[p_] == ']') { ++p_; break; }
                fail_("expected ',' or ']'");
            }
        } else if (c == '"') {
            v.kind = JsonValue::String;
            v.str = string_();
        } else if (lit_("true")) {
            v.kind = JsonValue::Bool; v.b = true;
        } else if (lit_("false")) {
            v.kind = JsonValue::Bool; v.b = false;
        } else if (lit_("null")) {
            v.kind = JsonValue::Null;
        } else if (lit_("NaN")) {
            v.kind = JsonValue::Number; v.num = std::strtod("nan", nullptr);
        } else {
            const char* b = s_.c_str() + p_;
            char* e = nullptr;
            double d = std::strtod(b, &e);
            if (e == b) fail_("unexpected token");
            p_ += static_cast<size_t>(e - b);
            v.kind = JsonValue::Number; v.num = d;
        }
        return v;
    }
    std::string string_() {
        std::string out;
        ++p_;  // opening quote
        while (p_ < s_.size() && s_[p_] != '"') {
            char c = s_[p_++];
            if (c != '\\') { out.push_back(c); continue; }
            if (p_ >= s_.size()) fail_("bad escape");
            char e = s_[p_++];
            switch (e) {
                case 'n': out.push_back('\n'); break;
                case 't': out.push_back('\t'); break;
                case 'r': out.push_back('\r'); break;
                case 'b': out.push_back('\b'); break;
                case 'f': out.push_back('\f'); break;
                case 'u': {
                    if (p_ + 4 > s_.size()) fail_("bad \\u escape");
                    unsigned cp = static_cast<unsigned>(std::strtoul(s_.substr(p_, 4).c_str(), nullptr, 16));
                    p_ += 4;
                    if (cp < 0x80) out.push_back(static_cast<char>(cp));
                    else if (cp < 0x800) { out.push_back(static_cast<char>(0xC0 | (cp >> 6))); out.push_back(static_cast<char>(0x80 | (cp & 0x3F))); }
                    else { out.push_back(static_cast<char>(0xE0 | (cp >> 12))); out.push_back(static_cast<char>(0x80 | ((cp >> 6) & 0x3F))); out.push_back(static_cast<char>(0x80 | (cp & 0x3F))); }
                    break;
                }
                default: out.push_back(e); break;  // \" \\ \/
            }
        }
        if (p_ >= s_.size()) fail_("unterminated string");
        ++p_;  // closing quote
        return out;
    }
};

inline JsonValue json_parse_file(const std::string& path) {
    std::string text = read_text_file(path);
    return JsonParser(text).parse();
}

// ----------------------------------------------------------------------------------------------
// .npy member view + uncompressed .npz archive
// ----------------------------------------------------------------------------------------------
struct NpyView {
    char byte_order = '<';   // '<', '>', '|', '='
    char type_code = 'f';    // f,i,u,b,S,U
    uint32_t word_size = 4;  // bytes per element (for 'U': characters)
    bool fortran_order = false;
    std::vector<uint64_t> shape;
    uint64_t num_elements = 0;
    const uint8_t* payload = nullptr;  // first element

    template <typename T>
    T get_as(uint64_t i) const {
        const uint8_t* p = payload + i * word_size;
        if (byte_order == '>') throw std::runtime_error("npy: big-endian arrays are not supported");
        switch (type_code) {
            case 'f':
                if (word_size == 4) { float v; memcpy(&v, p, 4); return static_cast<T>(v); }
                if (word_size == 8) { double v; memcpy(&v, p, 8); return static_cast<T>(v); }
                break;
            case 'i':
                if (word_size == 1) { int8_t v; memcpy(&v, p, 1); return static_cast<T>(v); }
                if (word_size == 2) { int16_t v; memcpy(&v, p, 2); return static_cast<T>(v); }
                if (word_size == 4) { int32_t v; memcpy(&v, p, 4); return static_cast<T>(v); }
                if (word_size == 8) { int64_t v; memcpy(&v, p, 8); return static_cast<T>(v); }
                break;
            case 'u':
            case 'b':
                if (word_size == 1) { uint8_t v; memcpy(&v, p, 1); return static_cast<T>(v); }
                if (word_size == 2) { uint16_t v; memcpy(&v, p, 2); return static_cast<T>(v); }
                if (word_size == 4) { uint32_t v; memcpy(&v, p, 4); return static_cast<T>(v); }
                if (word_size == 8) { uint64_t v; memcpy(&v, p, 8); return static_cast<T>(v); }
                break;
            default: break;
        }
        throw std::runtime_error("npy: unsupported dtype for numeric conversion");
    }

    // Bulk conversion into a caller-provided buffer (fast path when the dtype already matches).
    template <typename T>
    void copy_to(T* dst) const {
        const bool is_float_T = std::is_floating_point<T>::value;
        const bool same =
            (byte_order != '>') && word_size == sizeof(T) &&
            ((is_float_T && type_code == 'f') ||
             (!is_float_T && (type_code == 'u' || type_code == 'i')));  // non-negative ints: i == u bitwise
        if (same) { memcpy(dst, payload, num_elements * sizeof(T)); return; }
        for (uint64_t i = 0; i < num_elements; ++i) dst[i] = get_as<T>(i);
    }

    std::string as_text() const {  // for the 'format' member of scipy npz ("csc"/"csr"), dtype S or U
        std::string out;
        if (type_code == 'S') {
            for (uint64_t i = 0; i < word_size && payload[i]; ++i) out.push_back(static_cast<char>(payload[i]));
        } else if (type_code == 'U') {
            for (uint64_t i = 0; i < word_size; ++i) {
                uint32_t cp; memcpy(&cp, payload + 4 * i, 4);
                if (!cp) break;
                out.push_back(static_cast<char>(cp));
            }
        }
        return out;
    }
};

inline NpyView parse_npy(const uint8_t* p, uint64_t avail) {
    static const uint8_t magic[6] = {0x93, 'N', 'U', 'M', 'P', 'Y'};
    if (avail < 10 || memcmp(p, magic, 6) != 0) throw std::runtime_error("npy: bad magic");
    uint8_t major = p[6];
    uint64_t header_len, header_off;
    if (major == 1) { uint16_t h; memcpy(&h, p + 8, 2); header_len = h; header_off = 10; }
    else if (major == 2 || major == 3) { uint32_t h; memcpy(&h, p + 8, 4); header_len = h; header_off = 12; }
    else throw std::runtime_error("npy: unsupported major version");
    if (header_off + header_len > avail) throw std::runtime_error("npy: truncated header");
    std::string header(reinterpret_cast<const char*>(p + header_off), header_len);

    NpyView v;
    auto find_after = [&](const char* key) -> size_t {
        size_t k = header.find(key);
        if (k == std::string::npos) throw std::runtime_error(std::string("npy: header lacks ") + key);
        k = header.find(':', k);
        if (k == std::string::npos) throw std::runtime_error("npy: malformed header");
        return k + 1;
    };
    {   // descr
        size_t k = find_after("'descr'");
        size_t q0 = header.find('\'', k);
        size_t q1 = header.find('\'', q0 + 1);
        if (q0 == std::string::npos || q1 == std::string::npos) throw std::runtime_error("npy: malformed descr");
        std::string d = header.substr(q0 + 1, q1 - q0 - 1);
        if (d.size() < 3) throw std::runtime_error("npy: malformed descr '" + d + "'");
        v.byte_order = d[0];
        v.type_code = d[1];
        v.word_size = static_cast<uint32_t>(std::strtoul(d.c_str() + 2, nullptr, 10));
    }
    {   // fortran_order
        size_t k = find_after("'fortran_order'");
        while (k < header.size() && header[k] == ' ') ++k;
        v.fortran_order = header.compare(k, 4, "True") == 0;
    }
    {   // shape
        size_t k = find_after("'shape'");
        size_t a = header.find('(', k), b = header.find(')', k);
        if (a == std::string::npos || b == std::string::npos) throw std::runtime_error("npy: malformed shape");
        std::string s = header.substr(a + 1, b - a - 1);
        v.num_elements = 1;
        const char* c = s.c_str();
        while (*c) {
            while (*c == ' ' || *c == ',') ++c;
            if (!*c) break;
            char* e = nullptr;
            uint64_t dim = std::strtoull(c, &e, 10);
            if (e == c) break;
            v.shape.push_back(dim);
            v.num_elements *= dim;
            c = e;
        }
    }
    uint64_t elem_bytes = (v.type_code == 'U') ? 4ull * v.word_size : v.word_size;
    uint64_t payload_off = header_off + header_len;
    if (payload_off + v.num_elements * elem_bytes > avail) throw std::runtime_error("npy: truncated payload");
    v.payload = p + payload_off;
    if (v.type_code == 'U') { /* word_size counts UCS4 characters */ }
    return v;
}

// Uncompressed zip archive of .npy members (what numpy.savez / scipy.sparse.save_npz(compressed=False) write).
class NpzFile {
public:
    explicit NpzFile(const std::string& path) {
        file_.open(path, /*populate=*/false);
        index_();
    }
    bool has(const std::string& name) const { return members_.count(name) != 0; }
    NpyView get(const std::string& name) const {
        auto it = members_.find(name);
        if (it == members_.end()) throw std::runtime_error("npz: member '" + name + "' missing in " + file_.path());
        return parse_npy(file_.data() + it->second.first, it->second.second);
    }

private:
    MappedFile file_;
    std::map<std::string, std::pair<uint64_t, uint64_t>> members_;  // name (without .npy) -> (offset, size)

    template <typename T>
    T rd_(uint64_t off) const {
        if (off + sizeof(T) > file_.size()) throw std::runtime_error("npz: truncated archive " + file_.path());
        T v; memcpy(&v, file_.data() + off, sizeof(T)); return v;
    }

    void index_() {
        const uint8_t* d = file_.data();
        const uint64_t n = file_.size();
        if (n < 22) throw std::runtime_error("npz: file too small " + file_.path());
        // End-of-central-directory record: scan backwards for PK\5\6
        uint64_t eocd = UINT64_MAX;
        uint64_t lo = n > (22 + 65535) ? n - (22 + 65535) : 0;
        for (uint64_t i = n - 22 + 1; i-- > lo;) {
            if (d[i] == 'P' && d[i + 1] == 'K' && d[i + 2] == 5 && d[i + 3] == 6) { eocd = i; break; }
        }
        if (eocd == UINT64_MAX) throw std::runtime_error("npz: not a zip archive " + file_.path());
        uint64_t n_entries = rd_<uint16_t>(eocd + 10);
        uint64_t cd_size = rd_<uint32_t>(eocd + 12);
        uint64_t cd_off = rd_<uint32_t>(eocd + 16);
        if (n_entries == 0xFFFF || cd_size == 0xFFFFFFFFull || cd_off == 0xFFFFFFFFull) {
            // zip64: locator sits right before the EOCD
            if (eocd < 20) throw std::runtime_error("npz: bad zip64 locator");
            uint64_t loc = eocd - 20;
            if (rd_<uint32_t>(loc) != 0x07064b50u) throw std::runtime_error("npz: zip64 locator missing");
            uint64_t eocd64 = rd_<uint64_t>(loc + 8);
            if (rd_<uint32_t>(eocd64) != 0x06064b50u) throw std::runtime_error("npz: zip64 EOCD missing");
            n_entries = rd_<uint64_t>(eocd64 + 32);
            cd_size = rd_<uint64_t>(eocd64 + 40);
            cd_off = rd_<uint64_t>(eocd64 + 48);
        }
        (void)cd_size;
        uint64_t p = cd_off;
        for (uint64_t e = 0; e < n_entries; ++e) {
            if (rd_<uint32_t>(p) != 0x02014b50u) throw std::runtime_error("npz: bad central directory entry");
            uint16_t method = rd_<uint16_t>(p + 10);
            uint64_t csize = rd_<uint32_t>(p + 20);
            uint64_t usize = rd_<uint32_t>(p + 24);
            uint16_t name_len = rd_<uint16_t>(p + 28);
            uint16_t extra_len = rd_<uint16_t>(p + 30);
            uint16_t comment_len = rd_<uint16_t>(p + 32);
            uint64_t local_off = rd_<uint32_t>(p + 42);
            std::string name(reinterpret_cast<const char*>(d + p + 46), name_len);
            // zip64 extended information (header id 0x0001) carries the fields that overflowed, in order
            uint64_t x = p + 46 + name_len, x_end = x + extra_len;
            while (x + 4 <= x_end) {
                uint16_t id = rd_<uint16_t>(x), sz = rd_<uint16_t>(x + 2);
                if (id == 0x0001) {
                    uint64_t q = x + 4;
                    if (usize == 0xFFFFFFFFull) { usize = rd_<uint64_t>(q); q += 8; }
                    if (csize == 0xFFFFFFFFull) { csize = rd_<uint64_t>(q); q += 8; }
                    if (local_off == 0xFFFFFFFFull) { local_off = rd_<uint64_t>(q); q += 8; }
                }
                x += 4 + sz;
            }
            if (method != 0) {
                throw std::runtime_error("npz: member '" + name + "' of " + file_.path() +
                                         " is compressed; only uncompressed npz is supported (same as the reference loader)");
            }
            if (csize != usize) throw std::runtime_error("npz: stored member with csize != usize");
            // local header: the name/extra lengths there may differ from the central directory ones
            if (rd_<uint32_t>(local_off) != 0x04034b50u) throw std::runtime_error("npz: bad local header");
            uint16_t l_name = rd_<uint16_t>(local_off + 26), l_extra = rd_<uint16_t>(local_off + 28);
            uint64_t data_off = local_off + 30 + l_name + l_extra;
            if (data_off + usize > n) throw std::runtime_error("npz: member exceeds archive");
            if (name.size() > 4 && name.compare(name.size() - 4, 4, ".npy") == 0) name.resize(name.size() - 4);
            members_[name] = {data_off, usize};
            p += 46 + name_len + extra_len + comment_len;
        }
    }
};

// ----------------------------------------------------------------------------------------------
// PECOS mmap_store container (read side)
// ----------------------------------------------------------------------------------------------
class MmapStoreReader {
public:
    MmapStoreReader(const std::string& path, bool lazy_load) {
        file_.open(path, /*populate=*/!lazy_load);
        const uint8_t* d = file_.data();
        const uint64_t n = file_.size();
        if (n < 16) throw std::runtime_error("mmap_store: file too small " + path);
        static const uint8_t magic[6] = {0x93, 'P', 'E', 'C', 'O', 'S'};
        const uint8_t* sig = d + n - 16;
        if (memcmp(sig, magic, 6) != 0) throw std::runtime_error("File is not a valid PECOS MMAP file: " + path);
        if (sig[6] != '<') throw std::runtime_error("mmap_store: inconsistent endianness in " + path);
        if (sig[7] != 1) throw std::runtime_error("mmap_store: inconsistent version in " + path);
        uint64_t meta_off; memcpy(&meta_off, sig + 8, 8);
        if (meta_off + 8 > n) throw std::runtime_error("mmap_store: bad metadata offset in " + path);
        uint64_t n_blocks; memcpy(&n_blocks, d + meta_off, 8);
        if (meta_off + 8 + 16 * n_blocks > n) throw std::runtime_error("mmap_store: truncated metadata in " + path);
        blocks_.resize(n_blocks);
        for (uint64_t i = 0; i < n_blocks; ++i) {
            memcpy(&blocks_[i].first, d + meta_off + 8 + 16 * i, 8);
            memcpy(&blocks_[i].second, d + meta_off + 16 + 16 * i, 8);
            if (blocks_[i].first + blocks_[i].second > meta_off) throw std::runtime_error("mmap_store: block out of range in " + path);
        }
    }

    // Blocks are consumed strictly in the order they were written (mmap_util.hpp:113-117).
    template <typename T>
    const T* get_multiple(uint64_t n_elements) {
        if (next_ >= blocks_.size()) throw std::runtime_error("mmap_store: no more blocks in " + file_.path());
        auto blk = blocks_[next_++];
        if (n_elements * sizeof(T) != blk.second) {
            throw std::runtime_error("mmap_store: block holds " + std::to_string(blk.second) + " bytes, asked for " +
                                     std::to_string(n_elements * sizeof(T)) + " in " + file_.path());
        }
        return reinterpret_cast<const T*>(file_.data() + blk.first);
    }
    template <typename T>
    T get_one() { return *get_multiple<T>(1); }

    // MmapableVector<T>: a u64 size block followed by a data block (mmap_util.hpp:526-537)
    template <typename T>
    const T* get_vector(uint64_t* size_out) {
        uint64_t sz = get_one<uint64_t>();
        *size_out = sz;
        return get_multiple<T>(sz);
    }
    uint64_t blocks_left() const { return blocks_.size() - next_; }

private:
    MappedFile file_;
    std::vector<std::pair<uint64_t, uint64_t>> blocks_;  // (offset, size)
    uint64_t next_ = 0;
};

// ----------------------------------------------------------------------------------------------
// PECOS mmap_store container (write side; pecos/core/utils/mmap_util.hpp:54-140, :304-317)
// ----------------------------------------------------------------------------------------------
class MmapStoreWriter {
public:
    explicit MmapStoreWriter(const std::string& path) : path_(path) {
        f_ = std::fopen(path.c_str(), "wb");
        if (!f_) throw std::runtime_error("mmap_store: cannot open " + path + " for writing");
    }
    ~MmapStoreWriter() { if (f_) std::fclose(f_); }
    MmapStoreWriter(const MmapStoreWriter&) = delete;
    MmapStoreWriter& operator=(const MmapStoreWriter&) = delete;

    template <typename T>
    void put_multiple(const T* data, uint64_t n) {  // one block, padded to 16-byte alignment
        const uint64_t bytes = n * sizeof(T);
        blocks_.emplace_back(off_, bytes);
        if (bytes && std::fwrite(data, 1, bytes, f_) != bytes) throw std::runtime_error("mmap_store: short write to " + path_);
        off_ += bytes;
        static const char zeros[16] = {0};
        const uint64_t pad = (16 - off_ % 16) % 16;
        if (pad && std::fwrite(zeros, 1, pad, f_) != pad) throw std::runtime_error("mmap_store: short write to " + path_);
        off_ += pad;
    }
    template <typename T>
    void put_one(const T& v) { put_multiple<T>(&v, 1); }
    template <typename T>
    void put_vector(const T* data, uint64_t n) {  // MmapableVector<T>: size block + data block
        put_one<uint64_t>(n);
        put_multiple<T>(data, n);
    }
    void close() {  // metadata [n][(offset, size) x n] + 16-byte signature
        const uint64_t meta_off = off_, n = blocks_.size();
        std::fwrite(&n, 8, 1, f_);
        for (auto& b : blocks_) { std::fwrite(&b.first, 8, 1, f_); std::fwrite(&b.second, 8, 1, f_); }
        const uint8_t sig[8] = {0x93, 'P', 'E', 'C', 'O', 'S', '<', 1};
        std::fwrite(sig, 1, 8, f_);
        std::fwrite(&meta_off, 8, 1, f_);
        if (std::fclose(f_) != 0) { f_ = nullptr; throw std::runtime_error("mmap_store: cannot finish " + path_); }
        f_ = nullptr;
    }

private:
    std::string path_;
    std::FILE* f_ = nullptr;
    uint64_t off_ = 0;
    std::vector<std::pair<uint64_t, uint64_t>> blocks_;
};

// ----------------------------------------------------------------------------------------------
// tiny host thread pool for load-time work
// ----------------------------------------------------------------------------------------------
template <typename F>
inline void parallel_for_chunks(uint64_t n, F&& fn) {
    unsigned hw = std::thread::hardware_concurrency();
    unsigned nt = std::max(1u, std::min(hw ? hw : 1u, 64u));
    if (n < 64 || nt == 1) { for (uint64_t i = 0; i < n; ++i) fn(i); return; }
    std::atomic<uint64_t> next{0};
    std::vector<std::thread> pool;
    std::exception_ptr err = nullptr;
    std::atomic<bool> failed{false};
    for (unsigned t = 0; t < nt; ++t) {
        pool.emplace_back([&]() {
            try {
                for (;;) {
                    uint64_t i0 = next.fetch_add(16);
                    if (i0 >= n || failed.load()) break;
                    uint64_t i1 = std::min(n, i0 + 16);
                    for (uint64_t i = i0; i < i1; ++i) fn(i);
                }
            } catch (...) {
                if (!failed.exchange(true)) err = std::current_exception();
            }
        });
    }
    for (auto& th : pool) th.join();
    if (err) std::rethrow_exception(err);
}

}  // namespace pb200
