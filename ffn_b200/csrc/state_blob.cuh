// state_blob.cuh — the versioned blobs of ffn_trainer_get_state / _set_state and ffn_examples_get_state / _set_state.
// A blob is a fixed prefix (magic, version, the number of header words, the payload's bytes and the FNV-1a 64 checksum
// of everything after the prefix), the header words (int64; what the payload's meaning depends on, each with the name a
// refusal reports), then the payload: the object's sections back to back.  A blob arrives from a file, so `open` checks
// all of it on the host before the caller copies anything to the device.
#pragma once

#include <cstdint>
#include <cstring>
#include <string>
#include <vector>

#include "host.cuh"

namespace ffn {
namespace blob {

struct Prefix {
  uint64_t magic;
  uint32_t version;
  uint32_t n_words;
  uint64_t payload_bytes;
  uint64_t checksum;   // FNV-1a 64 of the header words and the payload
};
static_assert(sizeof(Prefix) == 32, "the blob prefix is 32 bytes");

inline uint64_t fnv1a64(const uint8_t* p, size_t n) {
  uint64_t h = 0xcbf29ce484222325ull;
  for (size_t i = 0; i < n; ++i) {
    h ^= p[i];
    h *= 0x100000001b3ull;
  }
  return h;
}

// The header words an object writes, and expects back, with their names.
struct Header {
  std::vector<int64_t> word;
  std::vector<std::string> name;
  void add(const std::string& n, int64_t v) {
    word.push_back(v);
    name.push_back(n);
  }
  void add3(const std::string& n, const int v[3]) {
    for (int d = 0; d < 3; ++d) add(n, v[d]);
  }
  void add_bits(const std::string& n, float v) {   // floats and doubles are compared bit for bit
    uint32_t b;
    std::memcpy(&b, &v, 4);
    add(n, b);
  }
  void add_bits(const std::string& n, double v) {
    int64_t b;
    std::memcpy(&b, &v, 8);
    add(n, b);
  }
};

// One payload section: `bytes` bytes at p, in device memory unless host.
struct Section {
  void* p;
  size_t bytes;
  bool host;
};

inline size_t payload_bytes(const std::vector<Section>& s) {
  size_t n = 0;
  for (const Section& x : s) n += x.bytes;
  return n;
}

// The cap / *n idiom: *n = the blob's size; writes it to out only when out is given and cap holds it.  Copies the
// device sections on cudaStreamPerThread, synchronises, then signs the blob.  Reads only.
inline int get(uint64_t magic, uint32_t version, const Header& h, const std::vector<Section>& secs, void* out,
               int64_t cap, int64_t* n) {
  if (!n) return fail("null n");
  const size_t pb = payload_bytes(secs), total = sizeof(Prefix) + h.word.size() * 8 + pb;
  *n = (int64_t)total;
  if (!out || cap < (int64_t)total) return 0;
  uint8_t* o = static_cast<uint8_t*>(out);
  Prefix pre{magic, version, (uint32_t)h.word.size(), pb, 0};
  std::memcpy(o + sizeof(Prefix), h.word.data(), h.word.size() * 8);
  size_t at = sizeof(Prefix) + h.word.size() * 8;
  for (const Section& s : secs) {
    if (s.host)
      std::memcpy(o + at, s.p, s.bytes);
    else if (s.bytes)
      CUDA_OK(cudaMemcpyAsync(o + at, s.p, s.bytes, cudaMemcpyDeviceToHost, cudaStreamPerThread));
    at += s.bytes;
  }
  CUDA_OK(cudaStreamSynchronize(cudaStreamPerThread));
  pre.checksum = fnv1a64(o + sizeof(Prefix), total - sizeof(Prefix));
  std::memcpy(o, &pre, sizeof(Prefix));
  return 0;
}

// Checks a blob's length, magic, version, checksum and header words against what this object writes (`what` names
// the object in the messages).  On success *payload points at the payload, laid out as secs.
inline int open(const void* in, int64_t n, uint64_t magic, uint32_t version, const Header& h,
                const std::vector<Section>& secs, const char* what, const uint8_t** payload) {
  if (!in) return fail("null state");
  const std::string w = what;
  if (n < (int64_t)sizeof(Prefix))
    return fail(w + " state of " + std::to_string(n) + " bytes is truncated: shorter than its prefix");
  const uint8_t* b = static_cast<const uint8_t*>(in);
  Prefix pre;
  std::memcpy(&pre, b, sizeof(Prefix));
  if (pre.magic != magic) return fail("not a " + w + " state (bad magic)");
  if (pre.version != version)
    return fail(w + " state version " + std::to_string(pre.version) + ", this library reads version " +
                std::to_string(version));
  const uint64_t want = (uint64_t)sizeof(Prefix) + (uint64_t)pre.n_words * 8 + pre.payload_bytes;
  if (pre.payload_bytes > (uint64_t)n || want != (uint64_t)n)
    return fail(w + " state of " + std::to_string(n) + " bytes, its prefix describes " + std::to_string(want) +
                ": truncated or padded");
  if (fnv1a64(b + sizeof(Prefix), (size_t)n - sizeof(Prefix)) != pre.checksum)
    return fail(w + " state checksum mismatch: the blob is corrupted");
  const int64_t* words = reinterpret_cast<const int64_t*>(b + sizeof(Prefix));
  for (size_t i = 0; i < std::min<size_t>(pre.n_words, h.word.size()); ++i) {
    int64_t v;
    std::memcpy(&v, words + i, 8);
    if (v != h.word[i])
      return fail(w + " state was saved with another " + h.name[i] + " (" + std::to_string(v) + ", here " +
                  std::to_string(h.word[i]) + ")");
  }
  if (pre.n_words != h.word.size())
    return fail(w + " state has " + std::to_string(pre.n_words) + " header words, expected " +
                std::to_string(h.word.size()));
  if (pre.payload_bytes != payload_bytes(secs))
    return fail(w + " state payload of " + std::to_string(pre.payload_bytes) + " bytes, expected " +
                std::to_string(payload_bytes(secs)));
  *payload = b + sizeof(Prefix) + h.word.size() * 8;
  return 0;
}

// Copies a checked payload into the sections, device sections on cudaStreamPerThread, and synchronises.
inline int put(const uint8_t* payload, const std::vector<Section>& secs) {
  size_t at = 0;
  for (const Section& s : secs) {
    if (s.host)
      std::memcpy(s.p, payload + at, s.bytes);
    else if (s.bytes)
      CUDA_OK(cudaMemcpyAsync(s.p, payload + at, s.bytes, cudaMemcpyHostToDevice, cudaStreamPerThread));
    at += s.bytes;
  }
  CUDA_OK(cudaStreamSynchronize(cudaStreamPerThread));
  return 0;
}

// The offset of section i in the payload.
inline size_t offset(const std::vector<Section>& secs, size_t i) {
  size_t at = 0;
  for (size_t k = 0; k < i; ++k) at += secs[k].bytes;
  return at;
}

}  // namespace blob
}  // namespace ffn
