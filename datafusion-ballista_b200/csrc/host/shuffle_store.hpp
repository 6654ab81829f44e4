// The executor's shuffle store: every stage's output, kept in HBM and keyed by (job, stage, out_partition) -- the
// identity create_shuffle_path resolves (ballista/core/src/execution_plans/mod.rs:66-99).  It owns the executor-side
// rules of Ballista's shuffle (DESIGN.md §2):
//  * a re-run of a map task replaces that task's earlier pieces (task retry): a piece is identified by its file_id (the
//    map task's input partition; < 0 for the un-partitioned writer) and src_rank (the executor that ran the task; -1
//    for a piece read from a file);
//  * pieces stored on this executor are appended; pieces installed from peers leave the partition's pieces
//    stable-sorted by (src_rank, file_id).  The reduce side reads rows in piece order;
//  * no entry is ever left without pieces, so an absent partition is one that no task wrote rows to;
//  * a cancelled or failed task leaves nothing behind; removing a job or a stage drops its partitions.
// Plain host bookkeeping under a mutex of its own: no CUDA calls, and nothing is called out while the lock is held.
// Callers that also hold b200_engine::mu take it first.
#pragma once
#include <algorithm>
#include <map>
#include <mutex>
#include <string>
#include <vector>

#include "device_mem.hpp"

namespace b200 {

// rows [r0, r1) of a batch
struct Piece {
  int64_t file_id;
  DevBatchPtr batch;
  int64_t r0, r1;
  int32_t src_rank = 0;               // which executor's map task produced it (exchange)
  std::vector<int64_t> str_bytes;     // per Utf8 column of the batch: character bytes of rows [r0, r1); empty = unknown
};
struct ShuffleKey {
  std::string job;
  int64_t stage;
  int64_t part;
  bool operator<(const ShuffleKey& o) const {
    if (job != o.job) return job < o.job;
    if (stage != o.stage) return stage < o.stage;
    return part < o.part;
  }
};
struct StoredPiece {
  int64_t part;
  Piece piece;
};

class ShuffleStore {
 public:
  // A map task's output for partition k: replaces the task's earlier piece there and is appended.  A piece without rows
  // is kept only with keep_empty (a file that holds no rows); otherwise the entry is dropped if nothing else is in it.
  void store(const ShuffleKey& k, Piece pc, bool keep_empty) {
    std::lock_guard<std::mutex> g(mu_);
    auto& v = map_[k];
    drop_task(v, pc.file_id, pc.src_rank);
    if (pc.r1 > pc.r0 || keep_empty) v.push_back(std::move(pc));
    else if (v.empty()) map_.erase(k);
  }
  // The un-partitioned writer (no file id): its piece becomes the partition's only piece, with or without rows.
  void replace_partition(const ShuffleKey& k, Piece pc) {
    std::lock_guard<std::mutex> g(mu_);
    auto& v = map_[k];
    v.clear();
    v.push_back(std::move(pc));
  }
  // Pieces that arrived from peers (or were placed by them), by partition: each replaces the earlier piece of the same
  // map task, then the partition's pieces are stable-sorted by (src_rank, file_id).
  void install(const std::string& job, int64_t stage, const std::map<int64_t, std::vector<Piece>>& arrivals) {
    std::lock_guard<std::mutex> g(mu_);
    for (auto& kv : arrivals) {
      if (kv.second.empty()) continue;
      auto& v = map_[ShuffleKey{job, stage, kv.first}];
      for (auto& pc : kv.second) {
        drop_task(v, pc.file_id, pc.src_rank);
        v.push_back(pc);
      }
      std::stable_sort(v.begin(), v.end(), [](const Piece& a, const Piece& b) { return a.src_rank != b.src_rank ? a.src_rank < b.src_rank : a.file_id < b.file_id; });
    }
  }

  // the pieces of partition k in reading order; none when it is absent
  std::vector<Piece> pieces(const ShuffleKey& k) const {
    std::lock_guard<std::mutex> g(mu_);
    auto it = map_.find(k);
    return it == map_.end() ? std::vector<Piece>() : it->second;
  }
  // rows of partition k; -1 when it is absent
  int64_t rows(const ShuffleKey& k) const {
    std::lock_guard<std::mutex> g(mu_);
    auto it = map_.find(k);
    if (it == map_.end()) return -1;
    int64_t n = 0;
    for (auto& p : it->second) n += p.r1 - p.r0;
    return n;
  }
  // one more than the highest partition of (job, stage) present; 0 when there is none
  int partitions(const std::string& job, int64_t stage) const {
    std::lock_guard<std::mutex> g(mu_);
    int mx = 0;
    for (auto& kv : map_)
      if (kv.first.job == job && kv.first.stage == stage) mx = std::max(mx, (int)kv.first.part + 1);
    return mx;
  }
  // the pieces executor `rank` produced for (job, stage), by partition and then in reading order
  std::vector<StoredPiece> of_rank(const std::string& job, int64_t stage, int32_t rank) const {
    std::lock_guard<std::mutex> g(mu_);
    std::vector<StoredPiece> out;
    for (auto& kv : map_)
      if (kv.first.job == job && kv.first.stage == stage)
        for (auto& pc : kv.second)
          if (pc.src_rank == rank) out.push_back(StoredPiece{kv.first.part, pc});
    return out;
  }

  // what a failed or cancelled map task of (job, stage) with this input partition stored on executor `rank`: its
  // pieces (file_id == input_partition), and the un-partitioned writer's piece of that partition (file_id < 0)
  void remove_task(const std::string& job, int64_t stage, int64_t input_partition, int32_t rank) {
    std::lock_guard<std::mutex> g(mu_);
    for (auto it = map_.begin(); it != map_.end();) {
      if (it->first.job == job && it->first.stage == stage) {
        auto& v = it->second;
        v.erase(std::remove_if(v.begin(), v.end(), [&](const Piece& pc) { return (pc.file_id == input_partition || (pc.file_id < 0 && it->first.part == input_partition)) && pc.src_rank == rank; }), v.end());
        if (v.empty()) {
          it = map_.erase(it);
          continue;
        }
      }
      ++it;
    }
  }
  // partitions of (job, stage) handed over to the executors that own them
  void remove_parts(const std::string& job, int64_t stage, const std::vector<int64_t>& parts) {
    std::lock_guard<std::mutex> g(mu_);
    for (int64_t p : parts) map_.erase(ShuffleKey{job, stage, p});
  }
  void remove_stage(const std::string& job, int64_t stage) {
    std::lock_guard<std::mutex> g(mu_);
    for (auto it = map_.begin(); it != map_.end();) {
      if (it->first.job == job && it->first.stage == stage) it = map_.erase(it);
      else ++it;
    }
  }
  // returns whether the store is empty afterwards
  bool remove_job(const std::string& job) {
    std::lock_guard<std::mutex> g(mu_);
    for (auto it = map_.begin(); it != map_.end();) {
      if (it->first.job == job) it = map_.erase(it);
      else ++it;
    }
    return map_.empty();
  }
  void remove_all() {
    std::lock_guard<std::mutex> g(mu_);
    map_.clear();
  }

 private:
  static void drop_task(std::vector<Piece>& v, int64_t file_id, int32_t src_rank) {
    v.erase(std::remove_if(v.begin(), v.end(), [&](const Piece& pc) { return pc.file_id == file_id && pc.src_rank == src_rank; }), v.end());
  }
  mutable std::mutex mu_;
  std::map<ShuffleKey, std::vector<Piece>> map_;
};

}  // namespace b200
