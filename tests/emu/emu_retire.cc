// emu_retire.cc -- the mention scan (filter.cuh mention_scan_kernel) and its plan (device.cu Device::scan_mentions) under
// the CPU SIMT emulator. TEST INFRASTRUCTURE ONLY (built by tests/emu/emu_retire.py into its own .so; never part of
// libzgpu.so). The emulator driver emu_main.cc is compiled into this translation unit unchanged. Added here: the plan
// over a snapshot's layout, the launches over host memory, and Store::mentioned as the answer to compare with.
#include "emu_main.cc"

#include "../../spicedb-kubeapi-proxy_b200/csrc/filter.cuh"

extern "C" {

// Store::mentioned: type `type`'s bitmap words (they cover the id extent). Returns their number (nothing is written
// past cap).
uint64_t emu_mention_host(void* h, int type, uint32_t* out, uint64_t cap) {
  Emu* e = static_cast<Emu*>(h);
  Store::IdBits bits;
  e->st.mentioned(&bits);
  const std::vector<uint32_t>& b = bits[static_cast<size_t>(type)];
  for (uint64_t i = 0; i < b.size() && i < cap; ++i) out[i] = b[i];
  return b.size();
}

// device.cu scan_mentions over host memory: of the resident arrays (count <= 1: e->h, merged by emu_merge_and_verify
// when the test did so), or of shard `rank` of `count` built from the store as a sharded handle's shard holds it.
// max_types: types per launch. out: every type's words back to back; word0[t]: type t's first word. Returns the
// words, 0 when cap is too small or nothing was published.
uint64_t emu_mention_device(void* h, uint32_t rank, uint32_t count, uint32_t grid, uint32_t max_types, uint32_t* out,
                            uint64_t cap, uint64_t* word0, uint64_t* launches) {
  Emu* e = static_cast<Emu*>(h);
  if (!e->published) return 0;
  HostSnapshot shard;
  const HostSnapshot* s = &e->h;
  if (count > 1) {
    shard = e->st.build(rank, count);
    s = &shard;
  }
  std::vector<MentionType> types;
  const uint64_t words = mention_types(e->sc, s->rels, s->cls, s->n_objects, &types);
  if (words > cap) return 0;
  std::vector<uint32_t> bits(words, 0xDEADBEEFu);  // every word is written by the kernel
  MentionPlan p{};
  p.row_ptr = s->row_ptr.data();
  p.rrow_ptr = s->rrow_ptr.data();
  p.bits = bits.data();
  *launches = 0;
  for (size_t at = 0; at < types.size(); at += max_types) {
    p.n_types = static_cast<uint32_t>(std::min<size_t>(max_types, types.size() - at));
    std::copy(types.begin() + at, types.begin() + at + p.n_types, p.type);
    zg_emu::launch(mention_scan_kernel, p, grid, 64, 0);
    ++*launches;
  }
  for (size_t t = 0; t < types.size(); ++t) word0[t] = types[t].word0;
  word0[types.size()] = words;
  std::copy(bits.begin(), bits.end(), out);
  return words;
}

}  // extern "C"
