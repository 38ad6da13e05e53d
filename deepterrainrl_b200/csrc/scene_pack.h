// deepterrainrl_b200 -- reader for `.trlpack` scene files (named f64 / i32 arrays; written by tools/pack_scene.py
// from the reference's arg file + JSON assets + Caffe HDF5 weights).
// Layout: "TRLPACK1", u32 record count, then {u32 name_len, name, u32 dtype (0 f64 | 1 i32), u64 count, payload}.
#pragma once
#include <cstdint>
#include <fstream>
#include <istream>
#include <ostream>
#include <string>
#include <unordered_map>
#include <vector>

namespace trl {

class ScenePack {
public:
    bool load(const std::string& path, std::string* err) {
        std::ifstream in(path, std::ios::binary);
        if (!in) { if (err) *err = "cannot open scene pack: " + path; return false; }
        return read(in, path, err);
    }
    // a pack from a stream positioned at its magic that holds nothing after it (the scene section of a checkpoint); `path` names it in
    // the messages
    bool read(std::istream& in, const std::string& path, std::string* err) {
        char magic[8];
        in.read(magic, 8);
        if (!in || std::string(magic, 8) != "TRLPACK1") { if (err) *err = "not a TRLPACK1 file: " + path; return false; }
        uint32_t count = 0;
        in.read(reinterpret_cast<char*>(&count), 4);
        // every length in the file is checked against what is left of it before anything is allocated
        const std::streampos body = in.tellg();
        in.seekg(0, std::ios::end);
        const uint64_t file_size = (uint64_t)in.tellg();
        in.seekg(body);
        auto remaining = [&]() { return file_size - (uint64_t)in.tellg(); };
        for (uint32_t r = 0; r < count && in; ++r) {
            uint32_t len = 0, dtype = 0;
            uint64_t n = 0;
            in.read(reinterpret_cast<char*>(&len), 4);
            if (!in || len > 256 || len > remaining()) { if (err) *err = "damaged scene pack (record name): " + path; return false; }
            std::string name(len, ' ');
            in.read(&name[0], len);
            in.read(reinterpret_cast<char*>(&dtype), 4);
            in.read(reinterpret_cast<char*>(&n), 8);
            if (!in || dtype > 1 || n > remaining() / (dtype == 1 ? 4 : 8)) {
                if (err) *err = "damaged scene pack (record '" + name + "' is longer than the file): " + path;
                return false;
            }
            order_.push_back(name);
            if (dtype == 1) {
                std::vector<int32_t>& v = ints_[name];
                v.resize(n);
                in.read(reinterpret_cast<char*>(v.data()), (std::streamsize)(n * 4));
            } else {
                std::vector<double>& v = reals_[name];
                v.resize(n);
                in.read(reinterpret_cast<char*>(v.data()), (std::streamsize)(n * 8));
            }
        }
        if (!in) { if (err) *err = "truncated scene pack: " + path; return false; }
        return true;
    }
    const std::vector<double>& f64(const std::string& name) const {
        static const std::vector<double> empty;
        auto it = reals_.find(name);
        return it == reals_.end() ? empty : it->second;
    }
    const std::vector<int32_t>& i32(const std::string& name) const {
        static const std::vector<int32_t> empty;
        auto it = ints_.find(name);
        return it == ints_.end() ? empty : it->second;
    }
    bool has(const std::string& name) const { return reals_.count(name) || ints_.count(name); }
    void set_f64(const std::string& name, std::vector<double> v) { if (!has(name)) order_.push_back(name); reals_[name] = std::move(v); }
    void set_i32(const std::string& name, std::vector<int32_t> v) { if (!has(name)) order_.push_back(name); ints_[name] = std::move(v); }
    bool save(const std::string& path, std::string* err) const {
        std::ofstream out(path, std::ios::binary);
        if (!out) { if (err) *err = "cannot write " + path; return false; }
        return write(out);
    }
    bool write(std::ostream& out) const {
        out.write("TRLPACK1", 8);
        uint32_t count = (uint32_t)order_.size();
        out.write(reinterpret_cast<const char*>(&count), 4);
        for (const std::string& name : order_) {
            uint32_t len = (uint32_t)name.size();
            out.write(reinterpret_cast<const char*>(&len), 4);
            out.write(name.data(), len);
            auto it = ints_.find(name);
            uint32_t dtype = it != ints_.end() ? 1 : 0;
            out.write(reinterpret_cast<const char*>(&dtype), 4);
            if (dtype == 1) {
                uint64_t n = it->second.size();
                out.write(reinterpret_cast<const char*>(&n), 8);
                out.write(reinterpret_cast<const char*>(it->second.data()), (std::streamsize)(n * 4));
            } else {
                const std::vector<double>& v = reals_.at(name);
                uint64_t n = v.size();
                out.write(reinterpret_cast<const char*>(&n), 8);
                out.write(reinterpret_cast<const char*>(v.data()), (std::streamsize)(n * 8));
            }
        }
        return (bool)out;
    }

private:
    std::unordered_map<std::string, std::vector<double>> reals_;
    std::unordered_map<std::string, std::vector<int32_t>> ints_;
    std::vector<std::string> order_;
};

}  // namespace trl
