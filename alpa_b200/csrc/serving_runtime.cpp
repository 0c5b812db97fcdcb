// Native serving runtime: KV-cache allocators and the per-iteration batch builders used by iteration-level
// (continuous) batching.
//
// Reference behaviour: examples/llm_serving/model/opt_model_1d.py -- the external `ft_mha` package provides
// init_cache_manager / can_allocate / prepare_inputs / free_cache around a 1-D token cache, and
// IterationLevelInputPool:547 builds a ragged 1-D token batch (new prompts first, then one token per running
// sequence).  Here the cache is one [slots, heads, D] tensor per layer, managed one of two ways:
//   KVCacheManager       every sequence owns a contiguous slot range sized for its maximum length, so the attention
//                        kernel addresses a sequence with (first_slot, context_len) and no block table.  Ranges come
//                        from a first-fit free list with coalescing on release.
//   PagedKVCacheManager  the slots form fixed-size blocks handed out as a sequence grows (lowest free index first), so
//                        a sequence holds only the blocks its tokens fill and any free block serves any sequence.  The
//                        attention kernel reads key j of a sequence through its block table:
//                        row = table[j / block_size] * block_size + j % block_size.
#include <pybind11/pybind11.h>
#include <pybind11/stl.h>

#include <algorithm>
#include <cstdint>
#include <climits>
#include <map>
#include <set>
#include <stdexcept>
#include <string>
#include <unordered_map>
#include <vector>

namespace py = pybind11;

namespace abserve {

struct SeqInfo {
  int64_t start = 0;     // first cache slot
  int64_t capacity = 0;  // slots reserved
  int64_t length = 0;    // tokens already written
};

class KVCacheManager {
 public:
  explicit KVCacheManager(int64_t num_slots) : num_slots_(num_slots) {
    if (num_slots <= 0) throw std::invalid_argument("cache needs at least one slot");
    free_[0] = num_slots;
  }

  int64_t num_slots() const { return num_slots_; }
  int64_t num_free() const {
    int64_t n = 0;
    for (auto& kv : free_) n += kv.second;
    return n;
  }
  int64_t largest_free_range() const {
    int64_t n = 0;
    for (auto& kv : free_) n = std::max(n, kv.second);
    return n;
  }
  int64_t num_sequences() const { return static_cast<int64_t>(seqs_.size()); }
  bool has(int64_t seq_id) const { return seqs_.count(seq_id) != 0; }

  // Would all of these reservations fit right now (first-fit, in the given order)?
  bool can_allocate(const std::vector<int64_t>& max_lens) const {
    std::map<int64_t, int64_t> f = free_;
    for (int64_t need : max_lens) {
      if (need <= 0) continue;
      bool ok = false;
      for (auto it = f.begin(); it != f.end(); ++it) {
        if (it->second >= need) {
          int64_t s = it->first, n = it->second;
          f.erase(it);
          if (n > need) f[s + need] = n - need;
          ok = true;
          break;
        }
      }
      if (!ok) return false;
    }
    return true;
  }

  int64_t allocate(int64_t seq_id, int64_t max_len) {
    if (max_len <= 0) throw std::invalid_argument("max_len must be positive");
    if (seqs_.count(seq_id)) throw std::invalid_argument("sequence " + std::to_string(seq_id) + " already has a cache range");
    for (auto it = free_.begin(); it != free_.end(); ++it) {
      if (it->second >= max_len) {
        int64_t s = it->first, n = it->second;
        free_.erase(it);
        if (n > max_len) free_[s + max_len] = n - max_len;
        seqs_[seq_id] = SeqInfo{s, max_len, 0};
        return s;
      }
    }
    throw std::runtime_error("KV cache exhausted: no free range of " + std::to_string(max_len) + " slots");
  }

  void release(int64_t seq_id) {
    auto it = seqs_.find(seq_id);
    if (it == seqs_.end()) throw std::invalid_argument("unknown sequence " + std::to_string(seq_id));
    int64_t s = it->second.start, n = it->second.capacity;
    seqs_.erase(it);
    auto nxt = free_.lower_bound(s);
    if (nxt != free_.end() && s + n == nxt->first) {  // merge with the following hole
      n += nxt->second;
      nxt = free_.erase(nxt);
    }
    if (nxt != free_.begin()) {  // merge with the preceding hole
      auto prv = std::prev(nxt);
      if (prv->first + prv->second == s) {
        prv->second += n;
        return;
      }
    }
    free_[s] = n;
  }

  const SeqInfo& info(int64_t seq_id) const {
    auto it = seqs_.find(seq_id);
    if (it == seqs_.end()) throw std::invalid_argument("unknown sequence " + std::to_string(seq_id));
    return it->second;
  }

  // Reserve the slots of `n` new tokens of a sequence; returns the first of them.
  int64_t append(int64_t seq_id, int64_t n) {
    auto it = seqs_.find(seq_id);
    if (it == seqs_.end()) throw std::invalid_argument("unknown sequence " + std::to_string(seq_id));
    SeqInfo& s = it->second;
    if (s.length + n > s.capacity)
      throw std::runtime_error("sequence " + std::to_string(seq_id) + " outgrew its cache range");
    int64_t first = s.start + s.length;
    s.length += n;
    return first;
  }

  // Build the device-side index arrays of one iteration.  Tokens are laid out prompts first (all tokens of each new
  // prompt), then one token per running sequence, then padding up to `batch_tokens`.  For every token:
  //   slot      cache row its K/V is written to (padding -> `pad_slot`, a scratch row)
  //   seq_start first cache row of its sequence
  //   ctx_len   number of cache rows it attends to, itself included (padding -> 0)
  //   position  position inside the sequence (0-based)
  py::dict prepare_inputs(const std::vector<int64_t>& prompt_ids, const std::vector<int64_t>& prompt_lens,
                          const std::vector<int64_t>& decode_ids, int64_t batch_tokens, int64_t pad_slot) {
    if (prompt_ids.size() != prompt_lens.size()) throw std::invalid_argument("prompt ids / lens differ in length");
    int64_t total = static_cast<int64_t>(decode_ids.size());
    for (int64_t l : prompt_lens) total += l;
    if (batch_tokens < total) throw std::invalid_argument("batch of " + std::to_string(total) + " tokens exceeds the token budget");
    std::vector<int64_t> slot(batch_tokens, pad_slot), position(batch_tokens, 0);
    std::vector<int32_t> seq_start(batch_tokens, 0), ctx_len(batch_tokens, 0);
    std::vector<int64_t> logit_index;
    int64_t t = 0;
    for (size_t i = 0; i < prompt_ids.size(); ++i) {
      int64_t n = prompt_lens[i];
      int64_t first = append(prompt_ids[i], n);
      const SeqInfo& s = info(prompt_ids[i]);
      for (int64_t j = 0; j < n; ++j, ++t) {
        slot[t] = first + j;
        seq_start[t] = static_cast<int32_t>(s.start);
        position[t] = first + j - s.start;
        ctx_len[t] = static_cast<int32_t>(position[t] + 1);
      }
      logit_index.push_back(t - 1);
    }
    for (int64_t id : decode_ids) {
      int64_t first = append(id, 1);
      const SeqInfo& s = info(id);
      slot[t] = first;
      seq_start[t] = static_cast<int32_t>(s.start);
      position[t] = first - s.start;
      ctx_len[t] = static_cast<int32_t>(position[t] + 1);
      logit_index.push_back(t);
      ++t;
    }
    py::dict out;
    out["slot"] = slot;
    out["seq_start"] = seq_start;
    out["ctx_len"] = ctx_len;
    out["position"] = position;
    out["logit_index"] = logit_index;
    out["num_tokens"] = total;
    return out;
  }

  std::vector<std::pair<int64_t, int64_t>> free_ranges() const {
    return std::vector<std::pair<int64_t, int64_t>>(free_.begin(), free_.end());
  }

 private:
  int64_t num_slots_;
  std::map<int64_t, int64_t> free_;  // start -> size, non-adjacent, sorted
  std::unordered_map<int64_t, SeqInfo> seqs_;
};

// Fixed-size blocks on demand.  A sequence is a list of blocks and a length; it takes a new block whenever its length
// crosses a block boundary and returns all of them when it is freed.
class PagedKVCacheManager {
 public:
  PagedKVCacheManager(int64_t num_blocks, int64_t block_size) : num_blocks_(num_blocks), block_size_(block_size) {
    if (num_blocks <= 0) throw std::invalid_argument("cache needs at least one block");
    if (num_blocks > INT32_MAX) throw std::invalid_argument("block ids must fit int32");
    if (block_size <= 0 || block_size > 1024 || (block_size & (block_size - 1)))
      throw std::invalid_argument("block_size must be a power of two up to 1024");
    for (int64_t b = 0; b < num_blocks; ++b) free_.insert(static_cast<int32_t>(b));
  }

  int64_t num_blocks() const { return num_blocks_; }
  int64_t block_size() const { return block_size_; }
  int64_t num_free_blocks() const { return static_cast<int64_t>(free_.size()); }
  int64_t num_sequences() const { return static_cast<int64_t>(seqs_.size()); }
  bool has(int64_t seq_id) const { return seqs_.count(seq_id) != 0; }

  void allocate(int64_t seq_id) {
    if (seqs_.count(seq_id)) throw std::invalid_argument("sequence " + std::to_string(seq_id) + " is already allocated");
    seqs_[seq_id];
  }

  void release(int64_t seq_id) {
    auto it = seqs_.find(seq_id);
    if (it == seqs_.end()) throw std::invalid_argument("unknown sequence " + std::to_string(seq_id));
    for (int32_t b : it->second.blocks) free_.insert(b);
    seqs_.erase(it);
  }

  // Blocks that `n` more tokens of the sequence would take (a sequence not allocated yet counts as empty).
  int64_t blocks_needed(int64_t seq_id, int64_t n) const {
    auto it = seqs_.find(seq_id);
    const int64_t len = it == seqs_.end() ? 0 : it->second.length;
    const int64_t have = it == seqs_.end() ? 0 : static_cast<int64_t>(it->second.blocks.size());
    return std::max<int64_t>(0, (len + n + block_size_ - 1) / block_size_ - have);
  }

  // Grow the sequence by `n` tokens, taking blocks as needed; returns the position of the first new token.  Nothing
  // changes when the free blocks do not suffice.
  int64_t append(int64_t seq_id, int64_t n) {
    if (n < 0) throw std::invalid_argument("cannot append a negative number of tokens");
    PagedSeq& s = get(seq_id);
    const int64_t need = blocks_needed(seq_id, n);
    if (need > num_free_blocks())
      throw std::runtime_error("KV cache exhausted: sequence " + std::to_string(seq_id) + " needs " +
                               std::to_string(need) + " blocks, " + std::to_string(num_free_blocks()) + " are free");
    for (int64_t i = 0; i < need; ++i) {
      s.blocks.push_back(*free_.begin());
      free_.erase(free_.begin());
    }
    const int64_t first = s.length;
    s.length += n;
    return first;
  }

  int64_t length(int64_t seq_id) const { return get(seq_id).length; }
  std::vector<int32_t> block_table(int64_t seq_id) const { return get(seq_id).blocks; }

  // The device-side index arrays of one iteration, laid out as KVCacheManager::prepare_inputs lays them out: prefill
  // entries first (prefill_lens[i] tokens of sequence prefill_ids[i]; a chunk continues the sequence's cached tokens,
  // so its positions start at the sequence's length), then one token per decoding sequence, then padding.  Sequence i
  // of the batch (prefills, then decodes) is row i of `block_table`, [N, max(max_blocks, longest list)] int32 padded
  // with 0, and its tokens' seq_start is i.  `slot` = block * block_size + offset of the token's position.
  // `logit_index` lists the last token of every prefill entry whose prefill_ends flag is set (all of them when the
  // flags are omitted) and every decode token.  A call that throws (an unknown or repeated sequence, too few free
  // blocks) changes nothing.
  py::dict prepare_inputs(const std::vector<int64_t>& prefill_ids, const std::vector<int64_t>& prefill_lens,
                          const std::vector<int64_t>& decode_ids, int64_t batch_tokens, int64_t pad_slot,
                          const std::vector<bool>& prefill_ends, int64_t max_blocks) {
    if (prefill_ids.size() != prefill_lens.size()) throw std::invalid_argument("prefill ids / lens differ in length");
    if (!prefill_ends.empty() && prefill_ends.size() != prefill_ids.size())
      throw std::invalid_argument("prefill ids / ends differ in length");
    int64_t total = static_cast<int64_t>(decode_ids.size());
    for (int64_t l : prefill_lens) {
      if (l <= 0) throw std::invalid_argument("a prefill entry needs at least one token");
      total += l;
    }
    if (batch_tokens < total) throw std::invalid_argument("batch of " + std::to_string(total) + " tokens exceeds the token budget");
    std::vector<int64_t> ids(prefill_ids), lens(prefill_lens);
    ids.insert(ids.end(), decode_ids.begin(), decode_ids.end());
    lens.insert(lens.end(), decode_ids.size(), 1);
    int64_t need = 0;
    std::unordered_map<int64_t, int> seen;
    for (size_t i = 0; i < ids.size(); ++i) {
      if (!has(ids[i])) throw std::invalid_argument("unknown sequence " + std::to_string(ids[i]));
      if (seen[ids[i]]++) throw std::invalid_argument("sequence " + std::to_string(ids[i]) + " appears twice in the batch");
      need += blocks_needed(ids[i], lens[i]);
    }
    if (need > num_free_blocks())
      throw std::runtime_error("KV cache exhausted: the batch needs " + std::to_string(need) + " blocks, " +
                               std::to_string(num_free_blocks()) + " are free");
    std::vector<int64_t> slot(batch_tokens, pad_slot), position(batch_tokens, 0);
    std::vector<int32_t> seq_start(batch_tokens, 0), ctx_len(batch_tokens, 0);
    std::vector<int64_t> logit_index;
    std::vector<std::vector<int32_t>> table;
    int64_t t = 0;
    for (size_t i = 0; i < ids.size(); ++i) {
      const int64_t first = append(ids[i], lens[i]);
      const PagedSeq& s = get(ids[i]);
      for (int64_t j = 0; j < lens[i]; ++j, ++t) {
        const int64_t pos = first + j;
        slot[t] = static_cast<int64_t>(s.blocks[pos / block_size_]) * block_size_ + pos % block_size_;
        seq_start[t] = static_cast<int32_t>(i);
        position[t] = pos;
        ctx_len[t] = static_cast<int32_t>(pos + 1);
      }
      const bool decode = i >= prefill_ids.size();
      if (decode || prefill_ends.empty() || prefill_ends[i]) logit_index.push_back(t - 1);
      table.push_back(s.blocks);
      max_blocks = std::max(max_blocks, static_cast<int64_t>(s.blocks.size()));
    }
    for (auto& row : table) row.resize(max_blocks, 0);
    py::dict out;
    out["slot"] = slot;
    out["seq_start"] = seq_start;
    out["ctx_len"] = ctx_len;
    out["position"] = position;
    out["logit_index"] = logit_index;
    out["block_table"] = table;
    out["num_tokens"] = total;
    return out;
  }

 private:
  struct PagedSeq {
    std::vector<int32_t> blocks;
    int64_t length = 0;  // tokens written
  };
  PagedSeq& get(int64_t seq_id) {
    auto it = seqs_.find(seq_id);
    if (it == seqs_.end()) throw std::invalid_argument("unknown sequence " + std::to_string(seq_id));
    return it->second;
  }
  const PagedSeq& get(int64_t seq_id) const { return const_cast<PagedKVCacheManager*>(this)->get(seq_id); }

  int64_t num_blocks_, block_size_;
  std::set<int32_t> free_;  // lowest index handed out first
  std::unordered_map<int64_t, PagedSeq> seqs_;
};

}  // namespace abserve

void bind_serving_runtime(py::module_& m) {
  using namespace abserve;
  py::class_<KVCacheManager>(m, "KVCacheManager")
      .def(py::init<int64_t>(), py::arg("num_slots"))
      .def_property_readonly("num_slots", &KVCacheManager::num_slots)
      .def_property_readonly("num_free", &KVCacheManager::num_free)
      .def_property_readonly("largest_free_range", &KVCacheManager::largest_free_range)
      .def_property_readonly("num_sequences", &KVCacheManager::num_sequences)
      .def("has", &KVCacheManager::has)
      .def("can_allocate", &KVCacheManager::can_allocate)
      .def("allocate", &KVCacheManager::allocate)
      .def("free", &KVCacheManager::release)
      .def("append", &KVCacheManager::append)
      .def("start", [](const KVCacheManager& c, int64_t id) { return c.info(id).start; })
      .def("length", [](const KVCacheManager& c, int64_t id) { return c.info(id).length; })
      .def("capacity", [](const KVCacheManager& c, int64_t id) { return c.info(id).capacity; })
      .def("free_ranges", &KVCacheManager::free_ranges)
      .def("prepare_inputs", &KVCacheManager::prepare_inputs, py::arg("prompt_ids"), py::arg("prompt_lens"),
           py::arg("decode_ids"), py::arg("batch_tokens"), py::arg("pad_slot"));
  py::class_<PagedKVCacheManager>(m, "PagedKVCacheManager")
      .def(py::init<int64_t, int64_t>(), py::arg("num_blocks"), py::arg("block_size"))
      .def_property_readonly("num_blocks", &PagedKVCacheManager::num_blocks)
      .def_property_readonly("block_size", &PagedKVCacheManager::block_size)
      .def_property_readonly("num_free_blocks", &PagedKVCacheManager::num_free_blocks)
      .def_property_readonly("num_sequences", &PagedKVCacheManager::num_sequences)
      .def("has", &PagedKVCacheManager::has)
      .def("allocate", &PagedKVCacheManager::allocate)
      .def("free", &PagedKVCacheManager::release)
      .def("append", &PagedKVCacheManager::append)
      .def("blocks_needed", &PagedKVCacheManager::blocks_needed)
      .def("length", &PagedKVCacheManager::length)
      .def("block_table", &PagedKVCacheManager::block_table)
      .def("prepare_inputs", &PagedKVCacheManager::prepare_inputs, py::arg("prefill_ids"), py::arg("prefill_lens"),
           py::arg("decode_ids"), py::arg("batch_tokens"), py::arg("pad_slot"),
           py::arg("prefill_ends") = std::vector<bool>(), py::arg("max_blocks") = 0);
}
