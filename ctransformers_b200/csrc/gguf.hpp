// GGUF container reader (host side, read-only, mmap-backed).
//
// Replaces, for this path, the reference's gguf_init_from_file + llama_model_loader
// (reference: models/ggml/ggml.c:19561-19800, models/ggml/llama.cpp:1182-1488).  Like the reference
// reader it accepts v1 (32-bit counts) and treats every later version as the v2 layout
// (ggml.c:19597-19610), honours general.alignment (default 32) and bounds-checks everything.
#pragma once
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <map>
#include <stdexcept>
#include <string>
#include <vector>

#include <fcntl.h>
#include <sys/mman.h>
#include <sys/stat.h>
#include <unistd.h>

namespace ctb {

enum GGMLType : uint32_t {
  T_F32 = 0, T_F16 = 1, T_Q4_0 = 2, T_Q4_1 = 3, T_Q5_0 = 6, T_Q5_1 = 7, T_Q8_0 = 8, T_Q8_1 = 9,
  T_Q2_K = 10, T_Q3_K = 11, T_Q4_K = 12, T_Q5_K = 13, T_Q6_K = 14, T_Q8_K = 15,
};

// elements per block / bytes per block (reference: ggml.c type_traits, ggml.c:1638-1808)
inline int type_block_elems(uint32_t t) {
  switch (t) {
    case T_F32: case T_F16: return 1;
    case T_Q4_0: case T_Q4_1: case T_Q5_0: case T_Q5_1: case T_Q8_0: case T_Q8_1: return 32;
    case T_Q2_K: case T_Q3_K: case T_Q4_K: case T_Q5_K: case T_Q6_K: case T_Q8_K: return 256;
  }
  return 0;
}
inline int type_block_bytes(uint32_t t) {
  switch (t) {
    case T_F32: return 4; case T_F16: return 2;
    case T_Q4_0: return 18; case T_Q4_1: return 20; case T_Q5_0: return 22; case T_Q5_1: return 24;
    case T_Q8_0: return 34; case T_Q8_1: return 36;
    case T_Q2_K: return 84; case T_Q3_K: return 110; case T_Q4_K: return 144; case T_Q5_K: return 176;
    case T_Q6_K: return 210; case T_Q8_K: return 292;
  }
  return 0;
}
inline const char* type_name(uint32_t t) {
  switch (t) {
    case T_F32: return "f32"; case T_F16: return "f16"; case T_Q4_0: return "q4_0"; case T_Q4_1: return "q4_1"; case T_Q5_0: return "q5_0";
    case T_Q5_1: return "q5_1"; case T_Q8_0: return "q8_0";
    case T_Q4_K: return "q4_K"; case T_Q5_K: return "q5_K"; case T_Q6_K: return "q6_K";
  }
  return "unsupported";
}

struct GGUFValue {
  uint32_t type = 0;          // gguf_type
  uint64_t u = 0;             // integer / bool payload
  double f = 0;               // float payload
  std::string s;              // string payload
  uint32_t arr_type = 0;      // element type for arrays
  uint64_t arr_n = 0;
  const uint8_t* arr_data = nullptr;        // raw element bytes for numeric arrays (inside the mapping)
  std::vector<std::string> arr_str;         // string arrays
};

struct GGUFTensor {
  std::string name;
  uint32_t n_dims = 0;
  uint64_t ne[4] = {1, 1, 1, 1};   // ne[0] is the contiguous (K) dimension
  uint32_t type = 0;
  uint64_t offset = 0;
  const uint8_t* data = nullptr;
  uint64_t nbytes = 0;
};

class GGUFFile {
 public:
  explicit GGUFFile(const std::string& path) {
    fd_ = ::open(path.c_str(), O_RDONLY);
    if (fd_ < 0) throw std::runtime_error("cannot open '" + path + "'");
    struct stat st;
    if (fstat(fd_, &st) != 0) throw std::runtime_error("cannot stat '" + path + "'");
    size_ = (size_t)st.st_size;
    base_ = (const uint8_t*)mmap(nullptr, size_, PROT_READ, MAP_PRIVATE, fd_, 0);
    if (base_ == MAP_FAILED) { base_ = nullptr; throw std::runtime_error("mmap failed for '" + path + "'"); }
    parse();
  }
  ~GGUFFile() {
    if (base_) munmap((void*)base_, size_);
    if (fd_ >= 0) ::close(fd_);
  }
  GGUFFile(const GGUFFile&) = delete;
  GGUFFile& operator=(const GGUFFile&) = delete;

  uint32_t version = 0;
  std::map<std::string, GGUFValue> kv;
  std::vector<GGUFTensor> tensors;

  const GGUFValue* find(const std::string& key) const {
    auto it = kv.find(key);
    return it == kv.end() ? nullptr : &it->second;
  }
  const GGUFTensor* tensor(const std::string& name) const {
    auto it = index_.find(name);
    return it == index_.end() ? nullptr : &tensors[it->second];
  }
  const GGUFTensor& need_tensor(const std::string& name) const {
    const GGUFTensor* t = tensor(name);
    if (!t) throw std::runtime_error("tensor '" + name + "' not found");
    return *t;
  }
  uint32_t need_u32(const std::string& key) const {
    const GGUFValue* v = find(key);
    if (!v) throw std::runtime_error("key not found in model: " + key);
    return (uint32_t)v->u;
  }
  uint32_t get_u32(const std::string& key, uint32_t dflt) const { const GGUFValue* v = find(key); return v ? (uint32_t)v->u : dflt; }
  float need_f32(const std::string& key) const {
    const GGUFValue* v = find(key);
    if (!v) throw std::runtime_error("key not found in model: " + key);
    return (float)v->f;
  }
  float get_f32(const std::string& key, float dflt) const { const GGUFValue* v = find(key); return v ? (float)v->f : dflt; }
  std::string need_str(const std::string& key) const {
    const GGUFValue* v = find(key);
    if (!v) throw std::runtime_error("key not found in model: " + key);
    return v->s;
  }

  // bytes of one element of a numeric value type (0: not one)
  static size_t scalar_size(uint32_t t) {
    switch (t) {
      case 0: case 1: case 7: return 1;   // u8 i8 bool
      case 2: case 3: return 2;           // u16 i16
      case 4: case 5: case 6: return 4;   // u32 i32 f32
      case 10: case 11: case 12: return 8;  // u64 i64 f64
    }
    return 0;
  }

 private:
  int fd_ = -1;
  const uint8_t* base_ = nullptr;
  size_t size_ = 0, pos_ = 0;
  std::map<std::string, size_t> index_;

  void need(size_t n) const { if (pos_ + n > size_ || pos_ + n < pos_) throw std::runtime_error("GGUF: truncated file"); }
  template <typename T> T rd() { need(sizeof(T)); T v; memcpy(&v, base_ + pos_, sizeof(T)); pos_ += sizeof(T); return v; }
  uint64_t rd_count() { return version == 1 ? (uint64_t)rd<uint32_t>() : rd<uint64_t>(); }
  std::string rd_str() {
    uint64_t n = rd_count();
    need(n);
    std::string s((const char*)base_ + pos_, (size_t)n);
    pos_ += n;
    return s;
  }
  void rd_scalar(uint32_t t, GGUFValue& v) {
    switch (t) {
      case 0: v.u = rd<uint8_t>(); v.f = (double)v.u; break;
      case 1: { int8_t x = rd<int8_t>(); v.u = (uint64_t)(int64_t)x; v.f = x; } break;
      case 2: v.u = rd<uint16_t>(); v.f = (double)v.u; break;
      case 3: { int16_t x = rd<int16_t>(); v.u = (uint64_t)(int64_t)x; v.f = x; } break;
      case 4: v.u = rd<uint32_t>(); v.f = (double)v.u; break;
      case 5: { int32_t x = rd<int32_t>(); v.u = (uint64_t)(int64_t)x; v.f = x; } break;
      case 6: { float x = rd<float>(); v.f = x; v.u = (uint64_t)x; } break;
      case 7: v.u = rd<uint8_t>() != 0; v.f = (double)v.u; break;
      case 10: v.u = rd<uint64_t>(); v.f = (double)v.u; break;
      case 11: { int64_t x = rd<int64_t>(); v.u = (uint64_t)x; v.f = (double)x; } break;
      case 12: { double x = rd<double>(); v.f = x; v.u = (uint64_t)x; } break;
      default: throw std::runtime_error("GGUF: bad value type");
    }
  }

  void parse() {
    if (rd<uint32_t>() != 0x46554747u) throw std::runtime_error("not a GGUF file (bad magic)");
    version = rd<uint32_t>();
    const uint64_t n_tensors = rd_count();
    const uint64_t n_kv = rd_count();
    for (uint64_t i = 0; i < n_kv; i++) {
      std::string key = rd_str();
      GGUFValue v;
      v.type = rd<uint32_t>();
      if (v.type == 8) {
        v.s = rd_str();
      } else if (v.type == 9) {
        v.arr_type = rd<uint32_t>();
        v.arr_n = rd_count();
        if (v.arr_type == 8) {
          v.arr_str.reserve((size_t)v.arr_n);
          for (uint64_t j = 0; j < v.arr_n; j++) v.arr_str.push_back(rd_str());
        } else {
          size_t es = scalar_size(v.arr_type);
          if (!es) throw std::runtime_error("GGUF: bad array element type");
          if (v.arr_n > (size_ - pos_) / es) throw std::runtime_error("GGUF: truncated file");   // (no 64-bit wrap in es * n)
          need(es * v.arr_n);
          v.arr_data = base_ + pos_;
          pos_ += es * v.arr_n;
        }
      } else {
        rd_scalar(v.type, v);
      }
      kv[key] = std::move(v);
    }
    tensors.resize((size_t)n_tensors);
    for (auto& t : tensors) {
      t.name = rd_str();
      t.n_dims = rd<uint32_t>();
      if (t.n_dims > 4) throw std::runtime_error("GGUF: tensor with more than 4 dims");
      for (uint32_t d = 0; d < t.n_dims; d++) t.ne[d] = rd_count();
      t.type = rd<uint32_t>();
      t.offset = rd<uint64_t>();
    }
    const uint64_t align = get_u32("general.alignment", 32);
    if (align == 0 || (align & (align - 1)) != 0) throw std::runtime_error("GGUF: general.alignment must be a power of two");
    const size_t data_start = (pos_ + align - 1) / align * align;
    if (data_start > size_) throw std::runtime_error("GGUF: truncated file");
    for (size_t i = 0; i < tensors.size(); i++) {
      auto& t = tensors[i];
      const int be = type_block_elems(t.type), bb = type_block_bytes(t.type);
      if (!be) throw std::runtime_error("GGUF: tensor '" + t.name + "' has unsupported type " + std::to_string(t.type));
      if (t.ne[0] % be) throw std::runtime_error("GGUF: tensor '" + t.name + "' row length not a multiple of its block size");
      // overflow-checked size: every factor is bounded by the file size before it is multiplied in
      uint64_t nbytes = t.ne[0] / be * (uint64_t)bb;
      for (int d = 1; d < 4; d++) {
        if (t.ne[d] != 0 && nbytes > (uint64_t)size_ / t.ne[d]) throw std::runtime_error("GGUF: tensor '" + t.name + "' data out of file bounds");
        nbytes *= t.ne[d];
      }
      t.nbytes = nbytes;
      if (t.offset > size_ - data_start || t.nbytes > size_ - data_start - t.offset) throw std::runtime_error("GGUF: tensor '" + t.name + "' data out of file bounds");
      t.data = base_ + data_start + t.offset;
      index_[t.name] = i;
    }
  }
};

}  // namespace ctb
