// mrhbm_keys.h -- the key slot format on the host as plain functions over bytes (no CUDA runtime calls, no ctx).
// A key slot is kb bytes.  u64 keys: kb = 8, the key little endian; it stands for its 8 big-endian bytes (SURVEY A.4),
// so numeric order is byte order.  String keys: kb = 28 / 60 / 124, the escaped key zero padded.
#pragma once
#include <algorithm>
#include <cstdint>
#include <cstring>
#include <string>
#include <vector>

#include "../../include/mrhbm.h"
#include "mrhbm_dev.cuh"  // fnv_lua_step, word_hash_step / word_hash_finish, mulhi_u64_u32: the device partitioners

namespace mrhbm {

constexpr size_t kU64SlotBytes = 8;

// Key slots are zero padded, so a key byte 0x00 cannot be stored as such.  Bytes 0x00 and 0x01 travel escaped --
// 0x00 -> 01 01, 0x01 -> 01 02 -- which keeps the bytewise order of the keys ("a" < "a\0" < "a\1" < "ab", SURVEY A.3)
// and is the identity for text.  Record slots and the host-side store of long keys hold keys in this form; the
// device partitioner hashes the unescaped bytes, the iterator unescapes.
inline size_t esc_size(const unsigned char* key, size_t n) {
  size_t e = n;
  for (size_t i = 0; i < n; i++) e += key[i] <= 1;
  return e;
}
// the escaped form of key[0..n) to dst (room for esc_size(key, n)), returns its length
inline size_t escape(const unsigned char* key, size_t n, unsigned char* dst) {
  size_t o = 0;
  for (size_t i = 0; i < n; i++) {
    if (key[i] <= 1) {
      dst[o++] = 1;
      dst[o++] = (unsigned char)(key[i] + 1);
    } else {
      dst[o++] = key[i];
    }
  }
  return o;
}
// out = the original bytes of the escaped key esc[0..n) (a lone trailing 0x01 stays as it is)
inline void unescape(const void* esc, size_t n, std::vector<unsigned char>& out) {
  const unsigned char* e = (const unsigned char*)esc;
  out.clear();
  for (size_t i = 0; i < n; i++) {
    if (e[i] == 1 && i + 1 < n)
      out.push_back((unsigned char)(e[++i] - 1));
    else
      out.push_back(e[i]);
  }
}
// the length of the escaped key a string slot holds: up to its zero padding
inline size_t slot_esc_len(const unsigned char* slot, size_t kb) { return strnlen((const char*)slot, kb); }

// u64 <-> its 8 big-endian bytes
inline uint64_t be64_load(const unsigned char* b) {
  uint64_t v = 0;
  for (int i = 0; i < 8; i++) v = (v << 8) | b[i];
  return v;
}
inline void be64_store(uint64_t v, unsigned char* b) {
  for (int i = 0; i < 8; i++) b[i] = (unsigned char)(v >> (56 - 8 * i));
}
inline uint64_t slot_u64(const unsigned char* slot) {
  uint64_t v;
  memcpy(&v, slot, 8);
  return v;
}

// out = the original bytes of the key in a slot
inline void slot_key(const unsigned char* slot, size_t kb, std::vector<unsigned char>& out) {
  if (kb == kU64SlotBytes) {
    out.resize(8);
    be64_store(slot_u64(slot), out.data());
  } else {
    unescape(slot, slot_esc_len(slot, kb), out);
  }
}

// key order of escaped keys: bytewise, a proper prefix first (escaping preserves the order of the original bytes)
inline int esc_cmp(const unsigned char* a, size_t na, const unsigned char* b, size_t nb) {
  const int c = memcmp(a, b, std::min(na, nb));
  return c ? (c < 0 ? -1 : 1) : (na > nb) - (na < nb);
}
// key order of two slots.  Escaped keys hold no 0x00, so a string slot's zero padding sorts below every key byte
// and whole slots compare as their escaped keys do.
inline int slot_cmp(const unsigned char* a, const unsigned char* b, size_t kb) {
  if (kb == kU64SlotBytes) {
    const uint64_t x = slot_u64(a), y = slot_u64(b);
    return x < y ? -1 : x != y;
  }
  return esc_cmp(a, kb, b, kb);
}

// The partition bin_of (mrhbm_dev.cuh) gives a string key, for the escaped key esc of any length: FNV-in-doubles over
// the ORIGINAL bytes (examples/WordCount/partitionfn.lua:8-16), the word hash over the little-endian words of the
// STORED bytes, or (range partitioner) bisect_right of the original bytes over the original splitters spl.
inline uint32_t host_partition(uint32_t partitioner, uint32_t P, const std::vector<std::string>& spl,
                               const std::string& esc) {
  if (partitioner == MRHBM_PART_RANGE || partitioner == MRHBM_PART_FNV_LUA) {
    std::vector<unsigned char> raw;
    unescape(esc.data(), esc.size(), raw);
    if (partitioner == MRHBM_PART_RANGE)
      return (uint32_t)(std::upper_bound(spl.begin(), spl.end(), std::string(raw.begin(), raw.end())) - spl.begin());
    uint32_t h = 2166136261u;
    for (unsigned char b : raw) h = fnv_lua_step(h, b);
    return h % P;
  }
  uint64_t h = kWordHashSeed;
  for (size_t i = 0; i < esc.size(); i += 4) {
    uint32_t w = 0;
    memcpy(&w, esc.data() + i, std::min<size_t>(4, esc.size() - i));
    h = word_hash_step(h, w);
  }
  return mulhi_u64_u32(word_hash_finish(h), P);
}

// The range partitioner's table image as the device reads it, spl_inv [P], spl_pre [n], spl_slot [n * kb] (strings
// only; RangeBinParams), from the n = P - 1 checked splitters spl (original bytes, non-decreasing; u64: 8 big-endian):
//   threshold t_i = the escaped splitter zero padded to the key slot, when it fits; else its first slot bytes plus one
//   as a big-endian number: a key that fits a slot is >= a longer splitter iff its slot is STRICTLY greater than the
//   splitter's first slot bytes (on equality the key is a proper prefix of it).  Then key >= s_i <=> slot >= t_i for
//   every key a slot holds.  A threshold that would pass all ones lies above every slot key: it and the (equal or
//   larger) splitters after it are left out of the device search (fin = the finite ones, spl_n) and stay zero.
//   u64 keys: t_i = the splitter; inv[p] of partition p = [s_{p-1}, s_p) (s_{-1} = 0, s_{P-1} = 2^64).
struct RangeTable {
  std::vector<unsigned char> image;
  uint32_t fin = 0;
};
inline RangeTable range_table(const std::vector<std::string>& spl, uint32_t P, size_t kb) {
  const size_t n = spl.size();
  RangeTable rt;
  rt.image.resize(16 * (size_t)P + 8 * n + (kb == kU64SlotBytes ? 0 : n * kb));
  unsigned char *inv = rt.image.data(), *pre = inv + 16 * (size_t)P, *slot = pre + 8 * n;
  auto put = [](unsigned char* at, uint64_t v) { memcpy(at, &v, 8); };
  if (kb == kU64SlotBytes) {
    auto s = [&](size_t i) { return be64_load((const unsigned char*)spl[i].data()); };
    for (uint32_t p = 0; p < P; p++) {
      const unsigned __int128 lo = p ? s(p - 1) : 0, hi = p < n ? (unsigned __int128)s(p) : (unsigned __int128)1 << 64;
      const unsigned __int128 w = hi - lo, f = w ? ~(unsigned __int128)0 / w : 0;
      put(inv + 16 * p, (uint64_t)(f >> 64));
      put(inv + 16 * p + 8, (uint64_t)f);
      if (p < n) put(pre + 8 * p, (uint64_t)hi);
    }
    rt.fin = (uint32_t)n;
    return rt;
  }
  std::vector<unsigned char> esc;
  for (size_t i = 0; i < n; i++) {
    const unsigned char* s = (const unsigned char*)spl[i].data();
    esc.resize(esc_size(s, spl[i].size()));
    escape(s, spl[i].size(), esc.data());
    unsigned char* t = slot + i * kb;
    memcpy(t, esc.data(), std::min(esc.size(), kb));
    if (esc.size() > kb) {  // + 1 in the last slot byte, carried
      size_t j = kb;
      while (j > 0 && t[j - 1] == 0xff) t[--j] = 0;
      if (j == 0) break;  // above every slot key, and so is every later splitter
      t[j - 1]++;
    }
    put(pre + 8 * i, be64_load(t));
    rt.fin = (uint32_t)i + 1;
  }
  return rt;
}

}  // namespace mrhbm
