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
//                        With prefix caching on, full blocks are indexed by their token ids and the exact token prefix
//                        before them, and a new sequence starts from the longest indexed chain matching its tokens.
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
// crosses a block boundary and drops its references to all of them when it is freed.
//
// Prefix caching (off by default; off, every block has one owner and allocation, outputs and errors are those of the
// plain allocator).  A block is free, in use (reference count >= 1) or cached-evictable (count 0, content indexed).
// Once an iteration has laid out all block_size rows of a block for writing, and the token ids of the sequence up to
// it are known (prepare_inputs' input_ids), the block is indexed under its token ids and the entry of the block before
// it: an entry's id is unique for the life of the manager, so a key names the exact token prefix, and evicting a block
// (which drops its entry) leaves every block chained through it unmatchable.  Lookups compare the parent id and the
// token ids exactly; the hash only picks candidates.  Only full blocks are shared, and a sequence never writes into a
// block before its length, so no shared or indexed row is ever handed out as a write slot (prepare_inputs checks it).
// Allocation takes uncached free blocks first (lowest index), then evicts cached blocks, least recently released first
// (a sequence releases its blocks last one first).
// A sequence's `namespace` (allocate / match_prefix) is the root of its chain: blocks are shared only between sequences
// of one namespace.  K/V depend on more than the tokens when a LoRA adapter is applied, so the pool passes the adapter's
// load id (never reused); namespace 0 is the base model and keeps the keys of a manager without namespaces.
class PagedKVCacheManager {
 public:
  PagedKVCacheManager(int64_t num_blocks, int64_t block_size, bool prefix_caching = false, int hash_bits = 64)
      : num_blocks_(num_blocks), block_size_(block_size), prefix_caching_(prefix_caching) {
    if (num_blocks <= 0) throw std::invalid_argument("cache needs at least one block");
    if (num_blocks > INT32_MAX) throw std::invalid_argument("block ids must fit int32");
    if (block_size <= 0 || block_size > 1024 || (block_size & (block_size - 1)))
      throw std::invalid_argument("block_size must be a power of two up to 1024");
    // hash_bits < 64 makes collisions likely; tests use it to show that a lookup never trusts the hash alone
    if (hash_bits < 1 || hash_bits > 64) throw std::invalid_argument("hash_bits must be in 1..64");
    hash_mask_ = hash_bits == 64 ? ~uint64_t{0} : (uint64_t{1} << hash_bits) - 1;
    for (int64_t b = 0; b < num_blocks; ++b) free_.insert(static_cast<int32_t>(b));
    refs_.assign(num_blocks, 0);
    entries_.resize(num_blocks);
  }

  int64_t num_blocks() const { return num_blocks_; }
  int64_t block_size() const { return block_size_; }
  bool prefix_caching() const { return prefix_caching_; }
  // uncached free blocks plus cached-evictable ones: both can be handed out
  int64_t num_free_blocks() const { return static_cast<int64_t>(free_.size() + evictable_.size()); }
  int64_t num_sequences() const { return static_cast<int64_t>(seqs_.size()); }
  int64_t num_cached_blocks() const { return static_cast<int64_t>(index_.size()); }
  int64_t num_evictable_blocks() const { return static_cast<int64_t>(evictable_.size()); }
  bool has(int64_t seq_id) const { return seqs_.count(seq_id) != 0; }
  int64_t ref_count(int64_t block) const {
    if (block < 0 || block >= num_blocks_) throw std::invalid_argument("block id out of range");
    return refs_[block];
  }
  bool is_cached(int64_t block) const {
    if (block < 0 || block >= num_blocks_) throw std::invalid_argument("block id out of range");
    return entries_[block].id != 0;
  }

  void allocate(int64_t seq_id, int64_t ns = 0) {
    if (seqs_.count(seq_id)) throw std::invalid_argument("sequence " + std::to_string(seq_id) + " is already allocated");
    const uint64_t root = chain_root(ns);
    seqs_[seq_id].chain = root;
  }

  void release(int64_t seq_id) {
    auto it = seqs_.find(seq_id);
    if (it == seqs_.end()) throw std::invalid_argument("unknown sequence " + std::to_string(seq_id));
    // last block first: of one sequence's cached blocks the tail is evicted first, so its prefix stays matchable longest
    const std::vector<int32_t>& blocks = it->second.blocks;
    for (auto r = blocks.rbegin(); r != blocks.rend(); ++r) {
      const int32_t b = *r;
      if (--refs_[b] > 0) continue;
      if (entries_[b].id != 0) {
        evict_tick_[b] = ++tick_;
        evictable_[tick_] = b;
      } else {
        free_.insert(b);
      }
    }
    seqs_.erase(it);
  }

  // Allocate `seq_id` with the longest chain of indexed blocks matching `token_ids`, taking a reference on each.
  // Returns the tokens hit: a multiple of block_size, at most ((len(token_ids) - 1) / block_size) * block_size so the
  // last token is always computed (its logits are needed, and it never writes into a shared block).
  int64_t match_prefix(int64_t seq_id, const std::vector<int64_t>& token_ids, int64_t ns = 0) {
    if (!prefix_caching_) throw std::invalid_argument("match_prefix needs a manager with prefix_caching=True");
    if (seqs_.count(seq_id)) throw std::invalid_argument("sequence " + std::to_string(seq_id) + " is already allocated");
    const int64_t n = static_cast<int64_t>(token_ids.size());
    const int64_t max_blocks = n > 0 ? (n - 1) / block_size_ : 0;
    std::vector<int32_t> hit;
    uint64_t parent = chain_root(ns);
    for (int64_t k = 0; k < max_blocks; ++k) {
      const int32_t b = lookup(parent, token_ids.data() + k * block_size_);
      if (b < 0) break;
      hit.push_back(b);
      parent = entries_[b].id;
    }
    PagedSeq& s = seqs_[seq_id];
    for (int32_t b : hit) {
      if (refs_[b]++ == 0) {
        auto t = evict_tick_.find(b);
        evictable_.erase(t->second);
        evict_tick_.erase(t);
      }
    }
    s.blocks = hit;
    s.length = static_cast<int64_t>(hit.size()) * block_size_;
    s.tokens.assign(token_ids.begin(), token_ids.begin() + s.length);
    s.chain = parent;
    s.chained = static_cast<int64_t>(hit.size());
    return s.length;
  }

  // Drop every index entry: cached blocks become plain free blocks.  Only with no live sequence.
  void reset_prefix_cache() {
    if (!seqs_.empty())
      throw std::runtime_error("reset_prefix_cache: " + std::to_string(seqs_.size()) + " sequences are live");
    for (auto& kv : evictable_) free_.insert(kv.second);
    evictable_.clear();
    evict_tick_.clear();
    for (auto& kv : index_) entries_[kv.second] = Entry{};
    index_.clear();
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
    check_writable(s);
    for (int64_t i = 0; i < need; ++i) s.blocks.push_back(take_block());
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
  // With prefix caching on, `input_ids` (the batch's token ids, at least one per laid-out token) lets the manager
  // index the blocks this iteration fills, and the result also holds, per prefill entry, `chunk_start` (its first
  // token's index in the batch), `chunk_len` and `chunk_pos` (its first token's position: the cached length).
  py::dict prepare_inputs(const std::vector<int64_t>& prefill_ids, const std::vector<int64_t>& prefill_lens,
                          const std::vector<int64_t>& decode_ids, int64_t batch_tokens, int64_t pad_slot,
                          const std::vector<bool>& prefill_ends, int64_t max_blocks,
                          const std::vector<int64_t>& input_ids) {
    if (prefill_ids.size() != prefill_lens.size()) throw std::invalid_argument("prefill ids / lens differ in length");
    if (!prefill_ends.empty() && prefill_ends.size() != prefill_ids.size())
      throw std::invalid_argument("prefill ids / ends differ in length");
    int64_t total = static_cast<int64_t>(decode_ids.size());
    for (int64_t l : prefill_lens) {
      if (l <= 0) throw std::invalid_argument("a prefill entry needs at least one token");
      total += l;
    }
    if (batch_tokens < total) throw std::invalid_argument("batch of " + std::to_string(total) + " tokens exceeds the token budget");
    if (!input_ids.empty() && static_cast<int64_t>(input_ids.size()) < total)
      throw std::invalid_argument("input_ids holds " + std::to_string(input_ids.size()) + " tokens, the batch " +
                                  std::to_string(total));
    std::vector<int64_t> ids(prefill_ids), lens(prefill_lens);
    ids.insert(ids.end(), decode_ids.begin(), decode_ids.end());
    lens.insert(lens.end(), decode_ids.size(), 1);
    int64_t need = 0;
    std::unordered_map<int64_t, int> seen;
    for (size_t i = 0; i < ids.size(); ++i) {
      if (!has(ids[i])) throw std::invalid_argument("unknown sequence " + std::to_string(ids[i]));
      if (seen[ids[i]]++) throw std::invalid_argument("sequence " + std::to_string(ids[i]) + " appears twice in the batch");
      need += blocks_needed(ids[i], lens[i]);
      check_writable(get(ids[i]));
    }
    if (need > num_free_blocks())
      throw std::runtime_error("KV cache exhausted: the batch needs " + std::to_string(need) + " blocks, " +
                               std::to_string(num_free_blocks()) + " are free");
    std::vector<int64_t> slot(batch_tokens, pad_slot), position(batch_tokens, 0);
    std::vector<int32_t> seq_start(batch_tokens, 0), ctx_len(batch_tokens, 0);
    std::vector<int64_t> logit_index;
    std::vector<int32_t> chunk_start, chunk_len, chunk_pos;
    std::vector<std::vector<int32_t>> table;
    int64_t t = 0;
    for (size_t i = 0; i < ids.size(); ++i) {
      const int64_t t0 = t;
      const int64_t first = append(ids[i], lens[i]);
      PagedSeq& s = get(ids[i]);
      for (int64_t j = 0; j < lens[i]; ++j, ++t) {
        const int64_t pos = first + j;
        slot[t] = static_cast<int64_t>(s.blocks[pos / block_size_]) * block_size_ + pos % block_size_;
        seq_start[t] = static_cast<int32_t>(i);
        position[t] = pos;
        ctx_len[t] = static_cast<int32_t>(pos + 1);
      }
      const bool decode = i >= prefill_ids.size();
      if (decode || prefill_ends.empty() || prefill_ends[i]) logit_index.push_back(t - 1);
      if (prefix_caching_) {
        if (!decode) {
          chunk_start.push_back(static_cast<int32_t>(t0));
          chunk_len.push_back(static_cast<int32_t>(lens[i]));
          chunk_pos.push_back(static_cast<int32_t>(first));
        }
        record_tokens(s, first, input_ids, t0, lens[i]);
      }
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
    if (prefix_caching_) {
      out["chunk_start"] = chunk_start;
      out["chunk_len"] = chunk_len;
      out["chunk_pos"] = chunk_pos;
    }
    return out;
  }

 private:
  struct PagedSeq {
    std::vector<int32_t> blocks;
    int64_t length = 0;           // tokens written
    std::vector<int64_t> tokens;  // token ids of positions [0, tokens.size()) (prefix caching)
    uint64_t chain = 0;           // index entry of the prefix made of blocks [0, chained), or the namespace's root
    int64_t chained = 0;
  };
  struct Entry {
    uint64_t id = 0;  // 0: not indexed
    uint64_t parent = 0;
    uint64_t hash = 0;
    std::vector<int64_t> tokens;
  };

  // The parent key of a namespace's first block.  Entry ids count up from 1 and never reach bit 63, so a root of
  // namespace > 0 is never an entry id; namespace 0 keeps the root 0.
  static uint64_t chain_root(int64_t ns) {
    if (ns < 0) throw std::invalid_argument("prefix cache namespace must be >= 0");
    return ns == 0 ? 0 : (uint64_t{1} << 63) | static_cast<uint64_t>(ns);
  }

  PagedSeq& get(int64_t seq_id) {
    auto it = seqs_.find(seq_id);
    if (it == seqs_.end()) throw std::invalid_argument("unknown sequence " + std::to_string(seq_id));
    return it->second;
  }
  const PagedSeq& get(int64_t seq_id) const { return const_cast<PagedKVCacheManager*>(this)->get(seq_id); }

  uint64_t hash_of(uint64_t parent, const int64_t* tok) const {
    uint64_t h = 1469598103934665603ull ^ (parent * 0x9E3779B97F4A7C15ull);
    for (int64_t i = 0; i < block_size_; ++i) {
      h ^= static_cast<uint64_t>(tok[i]) + 0x9E3779B97F4A7C15ull + (h << 6) + (h >> 2);
      h *= 1099511628211ull;
    }
    return h & hash_mask_;
  }
  // The indexed block of the full block `tok` after the prefix `parent`, or -1.
  int32_t lookup(uint64_t parent, const int64_t* tok) const {
    auto range = index_.equal_range(hash_of(parent, tok));
    for (auto it = range.first; it != range.second; ++it) {
      const Entry& e = entries_[it->second];
      if (e.parent == parent && std::equal(e.tokens.begin(), e.tokens.end(), tok)) return it->second;
    }
    return -1;
  }

  // Invariant of prefix caching: the next write of `s` lands in a block only it holds and no entry indexes.
  void check_writable(const PagedSeq& s) const {
    if (s.length % block_size_ == 0 || s.blocks.empty()) return;
    const int32_t b = s.blocks.back();
    if (refs_[b] != 1 || entries_[b].id != 0)
      throw std::logic_error("prefix cache invariant broken: block " + std::to_string(b) +
                             " is shared or indexed but would be written");
  }

  int32_t take_block() {
    int32_t b;
    if (!free_.empty()) {
      b = *free_.begin();
      free_.erase(free_.begin());
    } else {  // evict the least recently released cached block; blocks chained through it can no longer match
      auto it = evictable_.begin();
      b = it->second;
      evictable_.erase(it);
      evict_tick_.erase(b);
      unindex(b);
    }
    refs_[b] = 1;
    return b;
  }

  void unindex(int32_t b) {
    Entry& e = entries_[b];
    auto range = index_.equal_range(e.hash);
    for (auto it = range.first; it != range.second; ++it)
      if (it->second == b) {
        index_.erase(it);
        break;
      }
    e = Entry{};
  }

  // Note the token ids of positions [first, first + n) (batch tokens t0..) and index the blocks they complete.  Without
  // token ids (or after a gap) the sequence's later blocks stay unindexed.
  void record_tokens(PagedSeq& s, int64_t first, const std::vector<int64_t>& input_ids, int64_t t0, int64_t n) {
    if (input_ids.empty() || static_cast<int64_t>(s.tokens.size()) != first) return;
    s.tokens.insert(s.tokens.end(), input_ids.begin() + t0, input_ids.begin() + t0 + n);
    while (s.chained < s.length / block_size_ && s.chained * block_size_ + block_size_ <= (int64_t)s.tokens.size()) {
      const int64_t k = s.chained;
      const int64_t* tok = s.tokens.data() + k * block_size_;
      const int32_t b = s.blocks[k];
      const int32_t found = lookup(s.chain, tok);
      if (found >= 0) {  // the same content is already indexed (computed by another sequence): chain through it
        s.chain = entries_[found].id;
      } else if (entries_[b].id == 0) {
        Entry& e = entries_[b];
        e.id = ++next_entry_;
        e.parent = s.chain;
        e.hash = hash_of(s.chain, tok);
        e.tokens.assign(tok, tok + block_size_);
        index_.emplace(e.hash, b);
        s.chain = e.id;
      } else {
        s.chain = entries_[b].id;
      }
      ++s.chained;
    }
  }

  int64_t num_blocks_, block_size_;
  bool prefix_caching_;
  uint64_t hash_mask_ = ~uint64_t{0};
  std::set<int32_t> free_;                          // uncached free blocks, lowest index handed out first
  std::map<uint64_t, int32_t> evictable_;           // release tick -> cached block with no reference (LRU first)
  std::unordered_map<int32_t, uint64_t> evict_tick_;
  std::vector<int32_t> refs_;
  std::vector<Entry> entries_;                      // per block
  std::unordered_multimap<uint64_t, int32_t> index_;  // hash -> indexed block
  uint64_t tick_ = 0, next_entry_ = 0;
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
      .def(py::init<int64_t, int64_t, bool, int>(), py::arg("num_blocks"), py::arg("block_size"),
           py::arg("prefix_caching") = false, py::arg("hash_bits") = 64)
      .def_property_readonly("num_blocks", &PagedKVCacheManager::num_blocks)
      .def_property_readonly("block_size", &PagedKVCacheManager::block_size)
      .def_property_readonly("num_free_blocks", &PagedKVCacheManager::num_free_blocks)
      .def_property_readonly("num_sequences", &PagedKVCacheManager::num_sequences)
      .def("has", &PagedKVCacheManager::has)
      .def("allocate", &PagedKVCacheManager::allocate, py::arg("seq_id"), py::arg("namespace") = 0)
      .def("free", &PagedKVCacheManager::release)
      .def("append", &PagedKVCacheManager::append)
      .def("blocks_needed", &PagedKVCacheManager::blocks_needed)
      .def("length", &PagedKVCacheManager::length)
      .def("block_table", &PagedKVCacheManager::block_table)
      .def_property_readonly("prefix_caching", &PagedKVCacheManager::prefix_caching)
      .def_property_readonly("num_cached_blocks", &PagedKVCacheManager::num_cached_blocks)
      .def_property_readonly("num_evictable_blocks", &PagedKVCacheManager::num_evictable_blocks)
      .def("ref_count", &PagedKVCacheManager::ref_count)
      .def("is_cached", &PagedKVCacheManager::is_cached)
      .def("match_prefix", &PagedKVCacheManager::match_prefix, py::arg("seq_id"), py::arg("token_ids"),
           py::arg("namespace") = 0)
      .def("reset_prefix_cache", &PagedKVCacheManager::reset_prefix_cache)
      .def("prepare_inputs", &PagedKVCacheManager::prepare_inputs, py::arg("prefill_ids"), py::arg("prefill_lens"),
           py::arg("decode_ids"), py::arg("batch_tokens"), py::arg("pad_slot"),
           py::arg("prefill_ends") = std::vector<bool>(), py::arg("max_blocks") = 0,
           py::arg("input_ids") = std::vector<int64_t>());
}
