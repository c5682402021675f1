// NumPy .npy (format version 1.0) records — the container cuVS index files are made of.
//
// The reference serialises every scalar and every mdspan of an index through RAFT's numpy serializer
// (raft::serialize_scalar / raft::serialize_mdspan, used by cpp/src/neighbors/ivf_pq/ivf_pq_serialize.cuh:38-86,
// ivf_flat/ivf_flat_serialize.cuh:44-84, detail/cagra/cagra_serialize.cuh:45-84, ivf_list.cuh:108-133; the header builder is
// also called directly by cpp/include/cuvs/util/file_io.hpp:186-224).  RAFT is a third-party dependency that is absent from
// /root/reference (fetched by CPM: cpp/cmake/thirdparty/get_raft.cmake), so its record format is restated here from the
// published NPY 1.0 specification as RAFT emits it:
//   "\x93NUMPY" 0x01 0x00 <uint16 LE header_len> "{'descr': '<f4', 'fortran_order': False, 'shape': (3, 4)}" + spaces + "\n"
// with the preamble padded to a multiple of 64 bytes, followed by the raw little-endian data; a scalar is a 0-d array
// (shape "()"); dtype = byte-order char ('<' for multi-byte types, '|' for 1-byte types) + kind ('f', 'i', 'u') + item size;
// enums are written as their underlying integer type, bool as '|u1'.
// The reader accepts any NPY 1.0/2.0 record whose item size and element count match (so files written by NumPy itself or
// by other RAFT versions load as well).
#pragma once
#include "common.hpp"

#include <library_types.h>

#include <cstdint>
#include <cstdlib>
#include <cstring>
#include <istream>
#include <ostream>
#include <string>
#include <type_traits>
#include <vector>

namespace b200 {
namespace npy {

template <typename T>
inline std::string descr_of()
{
  using U = std::conditional_t<std::is_enum_v<T>, std::underlying_type<T>, std::common_type<T>>;
  using V = typename U::type;
  const char kind = std::is_floating_point_v<V> ? 'f' : ((std::is_signed_v<V> && !std::is_same_v<V, bool>) ? 'i' : 'u');
  std::string s;
  s += sizeof(V) > 1 ? '<' : '|';
  s += kind;
  s += std::to_string(sizeof(V));
  return s;
}

inline void write_header(std::ostream& os, const std::string& descr, const std::vector<int64_t>& shape)
{
  std::string sh = "(";
  for (size_t i = 0; i < shape.size(); ++i) {
    sh += std::to_string(shape[i]);
    if (shape.size() == 1) sh += ",";
    else if (i + 1 < shape.size()) sh += ", ";
  }
  sh += ")";
  std::string dict = "{'descr': '" + descr + "', 'fortran_order': False, 'shape': " + sh + "}";
  const size_t preamble = 6 + 2 + 2 + dict.size() + 1;
  const size_t pad      = 64 - preamble % 64;
  dict.append(pad, ' ');
  dict += '\n';
  const uint16_t hlen = static_cast<uint16_t>(dict.size());
  os.write("\x93NUMPY", 6);
  os.put(1);
  os.put(0);
  os.write(reinterpret_cast<const char*>(&hlen), 2);
  os.write(dict.data(), static_cast<std::streamsize>(dict.size()));
}

template <typename T>
inline void write_scalar(std::ostream& os, const T& v)
{
  write_header(os, descr_of<T>(), {});
  os.write(reinterpret_cast<const char*>(&v), sizeof(T));
}

template <typename T>
inline void write_array(std::ostream& os, const T* host, const std::vector<int64_t>& shape)
{
  write_header(os, descr_of<T>(), shape);
  int64_t n = 1;
  for (auto e : shape) n *= e;
  os.write(reinterpret_cast<const char*>(host), static_cast<std::streamsize>(n * sizeof(T)));
}

struct header {
  std::string descr;
  bool fortran = false;
  std::vector<int64_t> shape;
  int item_size() const { return std::atoi(descr.c_str() + 2); }
  int64_t count() const
  {
    int64_t n = 1;
    for (auto e : shape) n *= e;
    return n;
  }
};

inline header read_header(std::istream& is, const char* what)
{
  char magic[8];
  is.read(magic, 8);
  B2_EXPECTS(bool(is) && std::memcmp(magic, "\x93NUMPY", 6) == 0, "%s: not a cuVS index file (NPY record expected)", what);
  uint32_t hlen = 0;
  if (magic[6] == 1) {
    uint16_t h16 = 0;
    is.read(reinterpret_cast<char*>(&h16), 2);
    hlen = h16;
  } else {
    is.read(reinterpret_cast<char*>(&hlen), 4);
  }
  B2_EXPECTS(bool(is) && hlen > 0 && hlen < (1u << 20), "%s: corrupt NPY header", what);
  std::string dict(hlen, ' ');
  is.read(dict.data(), hlen);
  B2_EXPECTS(bool(is), "%s: truncated NPY header", what);
  header h;
  auto value_after = [&](const char* key) -> size_t {
    size_t p = dict.find(key);
    B2_EXPECTS(p != std::string::npos, "%s: NPY header lacks %s", what, key);
    p = dict.find(':', p);
    B2_EXPECTS(p != std::string::npos, "%s: corrupt NPY header", what);
    return p + 1;
  };
  size_t p = dict.find('\'', value_after("descr"));
  size_t e = dict.find('\'', p + 1);
  B2_EXPECTS(p != std::string::npos && e != std::string::npos && e - p - 1 >= 3, "%s: corrupt NPY descr", what);
  h.descr   = dict.substr(p + 1, e - p - 1);
  h.fortran = dict.compare(dict.find_first_not_of(' ', value_after("fortran_order")), 4, "True") == 0;
  p         = dict.find('(', value_after("shape"));
  e         = dict.find(')', p);
  B2_EXPECTS(p != std::string::npos && e != std::string::npos, "%s: corrupt NPY shape", what);
  int64_t cur = -1;
  for (size_t i = p + 1; i < e; ++i) {
    const char c = dict[i];
    if (c >= '0' && c <= '9') cur = (cur < 0 ? 0 : cur) * 10 + (c - '0');
    else if (cur >= 0) { h.shape.push_back(cur); cur = -1; }
  }
  if (cur >= 0) h.shape.push_back(cur);
  return h;
}

template <typename T>
inline T read_scalar(std::istream& is, const char* what)
{
  const header h = read_header(is, what);
  B2_EXPECTS(h.count() == 1 && h.item_size() == static_cast<int>(sizeof(T)), "%s: scalar of %zu bytes expected, found '%s'", what, sizeof(T),
             h.descr.c_str());
  T v;
  is.read(reinterpret_cast<char*>(&v), sizeof(T));
  B2_EXPECTS(bool(is), "%s: truncated file", what);
  return v;
}

/** Reads an array of exactly `count` elements of sizeof(T) bytes (any shape with that element count). */
template <typename T>
inline void read_array(std::istream& is, T* host, int64_t count, const char* what, std::vector<int64_t>* shape_out = nullptr)
{
  const header h = read_header(is, what);
  B2_EXPECTS(!h.fortran, "%s: fortran-order arrays are not supported", what);
  B2_EXPECTS(h.item_size() == static_cast<int>(sizeof(T)) && h.count() == count, "%s: %lld elements of %zu bytes expected, found %lld of '%s'", what,
             (long long)count, sizeof(T), (long long)h.count(), h.descr.c_str());
  is.read(reinterpret_cast<char*>(host), static_cast<std::streamsize>(count * sizeof(T)));
  B2_EXPECTS(bool(is), "%s: truncated file", what);
  if (shape_out) *shape_out = h.shape;
}

/**
 * The element types an index file can hold: the 4-byte tag in front of a CAGRA or IVF-Flat file (kind and size, the reader
 * dispatches on them: c/src/neighbors/cagra.cpp:881-899, ivf_flat.cpp:307-325), the NPY descr of its data records (float16
 * is kind 'e' in the tag and 'f' to NumPy), the cudaDataType of CAGRA's strided dataset record (dataset_serialize.hpp:83-99)
 * and the element size.
 */
struct file_dtype {
  DLDataType dl;
  const char* tag;  // three characters; written with the terminating zero
  const char* descr;
  cudaDataType cuda;
  int size;
};
inline const file_dtype kFileDtypes[] = {{{kDLFloat, 32, 1}, "<f4", "<f4", CUDA_R_32F, 4},
                                         {{kDLFloat, 16, 1}, "<e2", "<f2", CUDA_R_16F, 2},
                                         {{kDLInt, 8, 1}, "|i1", "|i1", CUDA_R_8I, 1},
                                         {{kDLUInt, 8, 1}, "|u1", "|u1", CUDA_R_8U, 1}};
inline const file_dtype& file_dtype_for(DLDataType t)
{
  for (const file_dtype& f : kFileDtypes)
    if (f.dl.code == t.code && f.dl.bits == t.bits) return f;
  B2_FAIL("index files hold float32, float16, int8 or uint8 rows (got dtype code %d, bits %d)", int(t.code), int(t.bits));
}
/** The type a tag or an NPY descr names: byte order '<', '|' or '=', then kind and item size; null when it is none of the
 *  four. */
inline const file_dtype* file_dtype_named(const std::string& s)
{
  if (s.size() < 3 || (s[0] != '<' && s[0] != '|' && s[0] != '=')) return nullptr;
  const char kind = s[1] == 'e' ? 'f' : s[1];
  const int size  = std::atoi(s.c_str() + 2);
  for (const file_dtype& f : kFileDtypes)
    if (f.descr[1] == kind && f.size == size) return &f;
  return nullptr;
}

/** Reads an array of exactly `count` elements of `item_size` bytes whatever their kind (float16 is '<f2' to NumPy and '<e2'
 * to RAFT), as raw bytes. */
inline void read_raw(std::istream& is, void* host, int64_t count, int item_size, const char* what)
{
  const header h = read_header(is, what);
  B2_EXPECTS(!h.fortran, "%s: fortran-order arrays are not supported", what);
  B2_EXPECTS(h.item_size() == item_size && h.count() == count, "%s: %lld elements of %d bytes expected, found %lld of '%s'", what,
             (long long)count, item_size, (long long)h.count(), h.descr.c_str());
  is.read(reinterpret_cast<char*>(host), static_cast<std::streamsize>(count * item_size));
  B2_EXPECTS(bool(is), "%s: truncated file", what);
}

}  // namespace npy
}  // namespace b200
