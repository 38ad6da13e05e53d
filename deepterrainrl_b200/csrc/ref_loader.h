// deepterrainrl_b200 -- native readers for the reference's own input formats, so a scene can be created straight from a
// DeepTerrainRL checkout without the Python packer:
//   * arg files / argv   `-key= value` tokens, `//` comments, first match wins      util/ArgParser.cpp:15-140
//   * JSON assets        characters, controllers, states, terrain, `_scale.txt`       (jsoncpp in the reference)
//   * Caffe HDF5 weights superblock v0, old-style groups, contiguous f64 datasets     learning/NeuralNet.cpp:571-587
// The result is the same set of named arrays a `.trlpack` holds (see tools/pack_scene.py), so both paths share
// fill_model() and can be compared record by record.
#pragma once
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <fstream>
#include <map>
#include <memory>
#include <sstream>
#include <stdexcept>
#include <string>
#include <vector>

#include "scene_pack.h"

namespace trl {

// ---------------------------------------------------------------------------------------------- minimal JSON
struct JValue {
    enum Type { Null, Bool, Num, Str, Arr, Obj } type = Null;
    double num = 0;
    bool b = false;
    std::string str;
    std::vector<JValue> arr;
    std::vector<std::pair<std::string, JValue>> obj;

    const JValue* get(const std::string& k) const {
        for (auto& kv : obj) if (kv.first == k) return &kv.second;
        return nullptr;
    }
    double number(const std::string& k, double dflt) const {
        const JValue* v = get(k);
        if (!v || v->type == Null) return dflt;
        if (v->type == Bool) return v->b ? 1.0 : 0.0;
        if (v->type != Num) throw std::runtime_error("json: '" + k + "' is not numeric");
        return v->num;
    }
    std::string string(const std::string& k, const std::string& dflt) const {
        const JValue* v = get(k);
        return (v && v->type == Str) ? v->str : dflt;
    }
};

class JParser {
public:
    explicit JParser(const std::string& text) : s_(text) {}
    JValue parse() {
        JValue v = value();
        ws();
        return v;
    }

private:
    const std::string& s_;
    size_t p_ = 0;
    void ws() {
        while (p_ < s_.size()) {
            char c = s_[p_];
            if (c == ' ' || c == '\t' || c == '\n' || c == '\r') ++p_;
            else if (c == '/' && p_ + 1 < s_.size() && s_[p_ + 1] == '/') { while (p_ < s_.size() && s_[p_] != '\n') ++p_; }
            else break;
        }
    }
    [[noreturn]] void fail(const char* what) { throw std::runtime_error(std::string("json: ") + what + " at offset " + std::to_string(p_)); }
    JValue value() {
        ws();
        if (p_ >= s_.size()) fail("unexpected end");
        char c = s_[p_];
        JValue v;
        if (c == '{') {
            v.type = JValue::Obj;
            ++p_;
            ws();
            if (s_[p_] == '}') { ++p_; return v; }
            for (;;) {
                ws();
                if (s_[p_] != '"') fail("expected key");
                std::string k = str();
                ws();
                if (s_[p_] != ':') fail("expected ':'");
                ++p_;
                v.obj.emplace_back(k, value());
                ws();
                if (s_[p_] == ',') { ++p_; continue; }
                if (s_[p_] == '}') { ++p_; break; }
                fail("expected ',' or '}'");
            }
        } else if (c == '[') {
            v.type = JValue::Arr;
            ++p_;
            ws();
            if (s_[p_] == ']') { ++p_; return v; }
            for (;;) {
                v.arr.push_back(value());
                ws();
                if (s_[p_] == ',') { ++p_; continue; }
                if (s_[p_] == ']') { ++p_; break; }
                fail("expected ',' or ']'");
            }
        } else if (c == '"') {
            v.type = JValue::Str;
            v.str = str();
        } else if (!s_.compare(p_, 4, "true")) { v.type = JValue::Bool; v.b = true; p_ += 4; }
        else if (!s_.compare(p_, 5, "false")) { v.type = JValue::Bool; v.b = false; p_ += 5; }
        else if (!s_.compare(p_, 4, "null")) { p_ += 4; }
        else {
            const char* beg = s_.c_str() + p_;
            char* end = nullptr;
            v.num = std::strtod(beg, &end);
            if (end == beg) fail("bad number");
            v.type = JValue::Num;
            p_ += (size_t)(end - beg);
        }
        return v;
    }
    std::string str() {
        std::string out;
        ++p_;
        while (p_ < s_.size() && s_[p_] != '"') {
            if (s_[p_] == '\\' && p_ + 1 < s_.size()) { ++p_; char e = s_[p_]; out += (e == 'n' ? '\n' : e == 't' ? '\t' : e); }
            else out += s_[p_];
            ++p_;
        }
        ++p_;
        return out;
    }
};

inline std::string read_text(const std::string& path) {
    std::ifstream f(path, std::ios::binary);
    if (!f) throw std::runtime_error("cannot open " + path);
    std::stringstream ss;
    ss << f.rdbuf();
    return ss.str();
}
inline JValue load_json(const std::string& path) {
    std::string text = read_text(path);
    return JParser(text).parse();
}

// ---------------------------------------------------------------------------------------------- argument list
class ArgList {
public:
    void append_args(int argc, const char* const* argv) { for (int i = 0; i < argc; ++i) toks_.push_back(argv[i]); }
    // cArgParser::AppendArgs(file): whitespace-separated tokens, `//` starts a comment that runs to the end of the line
    void append_file(const std::string& path) {
        std::string text = read_text(path);
        std::istringstream lines(text);
        std::string line;
        while (std::getline(lines, line)) {
            size_t c = line.find("//");
            if (c != std::string::npos) line.resize(c);
            std::istringstream ls(line);
            std::string t;
            while (ls >> t) toks_.push_back(t);
        }
    }
    bool find(const std::string& key, std::string* out) const {
        const std::string k = "-" + key + "=";
        for (size_t i = 0; i + 1 < toks_.size(); ++i)
            if (toks_[i] == k) {
                const std::string& v = toks_[i + 1];
                if (v.size() >= 2 && v.front() == '-' && v.back() == '=') return false;
                *out = v;
                return true;
            }
        return false;
    }
    std::string str(const std::string& key, const std::string& dflt) const { std::string v; return find(key, &v) ? v : dflt; }
    double num(const std::string& key, double dflt) const { std::string v; return find(key, &v) ? std::strtod(v.c_str(), nullptr) : dflt; }
    bool has(const std::string& key) const { std::string v; return find(key, &v); }

private:
    std::vector<std::string> toks_;
};

// ---------------------------------------------------------------------------------------------- minimal HDF5
// Enough of HDF5 to read Caffe's ToHDF5 output: superblock v0, symbol-table groups (TREE / HEAP / SNOD), v1 object
// headers, contiguous little-endian f64 datasets.  Returns {"/data/<layer>/<idx>": values}.
class H5Reader {
public:
    explicit H5Reader(const std::string& path) {
        std::ifstream f(path, std::ios::binary);
        if (!f) throw std::runtime_error("cannot open " + path);
        b_.assign(std::istreambuf_iterator<char>(f), std::istreambuf_iterator<char>());
        static const unsigned char sig[8] = {0x89, 'H', 'D', 'F', '\r', '\n', 0x1a, '\n'};
        if (b_.size() < 96 || std::memcmp(b_.data(), sig, 8) != 0) throw std::runtime_error("not an HDF5 file: " + path);
        if (b_[8] != 0 || b_[13] != 8 || b_[14] != 8) throw std::runtime_error("unsupported HDF5 superblock: " + path);
        Entry root = ste(24 + 32);
        walk(root, "");
    }
    const std::map<std::string, std::vector<double>>& datasets() const { return out_; }

private:
    struct Entry { uint64_t name_off = 0, ohdr = 0, btree = 0, heap = 0; bool group = false; };
    std::vector<char> b_;
    std::map<std::string, std::vector<double>> out_;
    // every address and length below comes from the file: nothing is dereferenced before it has been checked against the image
    void need(uint64_t p, uint64_t n) const {
        if (p > b_.size() || n > b_.size() - p) throw std::runtime_error("hdf5: address past the end of the file");
    }
    bool tag(uint64_t p, const char* t4) const { need(p, 4); return std::memcmp(b_.data() + p, t4, 4) == 0; }
    template <typename T> T rd(uint64_t p) const {
        if (p > b_.size() || sizeof(T) > b_.size() - p) throw std::runtime_error("hdf5: read past end");
        T v;
        std::memcpy(&v, b_.data() + p, sizeof(T));
        return v;
    }
    Entry ste(uint64_t p) const {
        Entry e;
        e.name_off = rd<uint64_t>(p); e.ohdr = rd<uint64_t>(p + 8);
        if (rd<uint32_t>(p + 16) == 1) { e.group = true; e.btree = rd<uint64_t>(p + 24); e.heap = rd<uint64_t>(p + 32); }
        return e;
    }
    struct Msg { uint16_t type; uint64_t body; uint16_t size; };
    std::vector<Msg> messages(uint64_t addr) const {
        if (rd<uint8_t>(addr) != 1) throw std::runtime_error("hdf5: object header version");
        uint16_t nmsg = rd<uint16_t>(addr + 2);
        uint32_t hsize = rd<uint32_t>(addr + 8);
        std::vector<Msg> msgs;
        std::vector<std::pair<uint64_t, uint64_t>> blocks{{addr + 16, hsize}};
        for (size_t bi = 0; bi < blocks.size() && msgs.size() < nmsg; ++bi) {
            uint64_t p = blocks[bi].first, end = p + blocks[bi].second;
            while (p + 8 <= end && msgs.size() < nmsg) {
                Msg m{rd<uint16_t>(p), p + 8, rd<uint16_t>(p + 2)};
                if (m.type == 0x10) blocks.emplace_back(rd<uint64_t>(m.body), rd<uint64_t>(m.body + 8));
                msgs.push_back(m);
                p = m.body + m.size;
            }
        }
        return msgs;
    }
    void leaves(uint64_t addr, std::vector<uint64_t>& out, int depth = 0) const {
        if (depth > 16 || out.size() > 65536) throw std::runtime_error("hdf5: B-tree too deep / too wide (damaged file?)");
        if (!tag(addr, "TREE")) throw std::runtime_error("hdf5: bad B-tree node");
        uint8_t level = rd<uint8_t>(addr + 5);
        uint16_t n = rd<uint16_t>(addr + 6);
        uint64_t p = addr + 8 + 16 + 8;
        for (uint16_t i = 0; i < n; ++i) {
            uint64_t child = rd<uint64_t>(p);
            p += 16;
            if (level > 0) leaves(child, out, depth + 1); else out.push_back(child);
        }
    }
    void walk(Entry e, const std::string& prefix, int depth = 0) {
        if (depth > 8) throw std::runtime_error("hdf5: group nesting too deep (damaged file?)");
        if (!e.group)
            for (auto& m : messages(e.ohdr))
                if (m.type == 0x11) { e.group = true; e.btree = rd<uint64_t>(m.body); e.heap = rd<uint64_t>(m.body + 8); }
        if (e.group) {
            if (!tag(e.heap, "HEAP")) throw std::runtime_error("hdf5: bad local heap");
            uint64_t heap_data = rd<uint64_t>(e.heap + 24);
            std::vector<uint64_t> nodes;
            leaves(e.btree, nodes);
            for (uint64_t snod : nodes) {
                if (!tag(snod, "SNOD")) throw std::runtime_error("hdf5: bad symbol node");
                uint16_t n = rd<uint16_t>(snod + 6);
                for (uint16_t i = 0; i < n; ++i) {
                    Entry c = ste(snod + 8 + 40ull * i);
                    need(heap_data, c.name_off);
                    const uint64_t np = heap_data + c.name_off;
                    need(np, 1);
                    const void* nul = std::memchr(b_.data() + np, 0, b_.size() - np);
                    if (!nul || (const char*)nul - (b_.data() + np) > 255) throw std::runtime_error("hdf5: unterminated link name");
                    std::string name(b_.data() + np);
                    walk(c, prefix + "/" + name, depth + 1);
                }
            }
            return;
        }
        uint64_t count = 1, addr = 0, size = 0;
        for (auto& m : messages(e.ohdr)) {
            if (m.type == 0x1) {
                uint8_t ver = rd<uint8_t>(m.body), rank = rd<uint8_t>(m.body + 1);
                uint64_t p = m.body + (ver == 1 ? 8 : 4);
                count = 1;
                for (uint8_t r = 0; r < rank; ++r) {
                    const uint64_t dim = rd<uint64_t>(p + 8ull * r);
                    if (dim != 0 && count > b_.size() / dim) throw std::runtime_error("hdf5: dataspace larger than the file at " + prefix);
                    count *= dim;
                }
            } else if (m.type == 0x3) {
                if ((rd<uint8_t>(m.body) & 0x0f) != 1 || rd<uint32_t>(m.body + 4) != 8) throw std::runtime_error("hdf5: only f64 datasets are supported");
            } else if (m.type == 0x8) {
                if (rd<uint8_t>(m.body) != 3 || rd<uint8_t>(m.body + 1) != 1) throw std::runtime_error("hdf5: only contiguous v3 layouts are supported");
                addr = rd<uint64_t>(m.body + 2); size = rd<uint64_t>(m.body + 10);
            }
        }
        if (count > b_.size() / 8 || size != count * 8) throw std::runtime_error("hdf5: dataset size mismatch at " + prefix);
        need(addr, size);
        std::vector<double> v(count);
        std::memcpy(v.data(), b_.data() + addr, count * 8);
        out_[prefix] = std::move(v);
    }
};

// Builds the named arrays of a scene from reference-format inputs; `root` is the directory the relative paths in the
// arg file refer to (the DeepTerrainRL checkout).  Mirrors tools/pack_scene.py record for record.
void build_scene_from_args(int argc, const char* const* argv, const std::string& root, ScenePack* out);

// The records of a character file (`-character_file`) as the scene pack stores them: joints [nj][7], bodies [nj][9], pd [nj][6], the
// parameter sets of the controller files its Controllers section names (resolved against `root`, read for the raptor's layout when
// `raptor`) [n_ctrl][n_params], actions [n_actions][4], and the Controllers flags.  Throws on a malformed file, and (expect_nj >= 0)
// on a joint count other than expect_nj before any controller file is read.
struct CharacterRecords {
    int nj = 0, ndof = 0, n_ctrl = 0, n_actions = 0, default_action = 0, grav_comp = 1, virt_forces = 1;
    std::vector<double> joints, bodies, pd, ctrl_params, actions;
};
CharacterRecords read_character_file(const std::string& path, const std::string& root, bool raptor, int expect_nj = -1);
// path relative to root (absolute paths as given)
std::string join_path(const std::string& root, const std::string& rel);

// A terrain file (`-terrain_file`, cTerrainGen2D::LoadParams: {"Type": ..., "Params": [{...}, ...]}): the generator type and
// n_sets parameter sets of 40 each, every parameter a file does not name at its cTerrainGen2D default.  Throws on an unknown type
// or a malformed file.
struct TerrainFile {
    int type = 0;
    int n_sets = 0;
    std::vector<double> params;      // [n_sets][40]
};
TerrainFile read_terrain_file(const std::string& path);

}  // namespace trl
