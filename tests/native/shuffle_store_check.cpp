// CPU check of the shuffle store's rules (csrc/host/shuffle_store.hpp): task retry, piece order, the empty-partition
// outcomes, the cleanup of a failed task, stage and job removal, the partition count, one executor's snapshot and the
// hand-over of exchanged partitions.  Pieces carry batches without columns: the store never looks inside them.
#include <cstdio>
#include <string>
#include <vector>

#include "../../datafusion-ballista_b200/csrc/host/shuffle_store.hpp"

using namespace b200;

static int fails = 0;
#define CHECK(cond)                                                \
  do {                                                             \
    if (!(cond)) {                                                 \
      fails++;                                                     \
      printf("FAIL line %d: %s\n", __LINE__, #cond);               \
    }                                                              \
  } while (0)

static Piece piece(int64_t file_id, int32_t rank, int64_t rows) {
  auto b = std::make_shared<DevBatch>();
  b->n = rows;
  return Piece{file_id, b, 0, rows, rank, {}};
}
static ShuffleKey key(int64_t stage, int64_t part, const std::string& job = "j") { return ShuffleKey{job, stage, part}; }
// (src_rank, file_id, rows) of every piece, in reading order
static std::vector<std::vector<int64_t>> ids(const std::vector<Piece>& v) {
  std::vector<std::vector<int64_t>> o;
  for (auto& p : v) o.push_back({p.src_rank, p.file_id, p.r1 - p.r0});
  return o;
}
typedef std::vector<std::vector<int64_t>> Ids;

int main() {
  {  // task retry: the same map task (file_id, src_rank) replaces its piece; another executor's task of that id stays
    ShuffleStore s;
    s.store(key(1, 0), piece(3, 0, 10), false);
    s.store(key(1, 0), piece(4, 0, 2), false);
    s.store(key(1, 0), piece(3, 0, 5), false);
    CHECK(ids(s.pieces(key(1, 0))) == (Ids{{0, 4, 2}, {0, 3, 5}}));
    s.store(key(1, 0), piece(3, 1, 7), false);
    CHECK(s.rows(key(1, 0)) == 14);
    s.store(ShuffleKey{"j", 1, 0}, piece(3, -1, 1), true);  // a file's piece of the same map task id
    CHECK(ids(s.pieces(key(1, 0))) == (Ids{{0, 4, 2}, {0, 3, 5}, {1, 3, 7}, {-1, 3, 1}}));
    s.store(key(1, 0), piece(3, -1, 6), true);
    CHECK(ids(s.pieces(key(1, 0))) == (Ids{{0, 4, 2}, {0, 3, 5}, {1, 3, 7}, {-1, 3, 6}}));
  }
  {  // local pieces are appended; pieces installed from peers leave the partition sorted by (src_rank, file_id)
    ShuffleStore s;
    s.store(key(1, 0), piece(5, 1, 1), false);
    s.store(key(1, 0), piece(2, 0, 1), false);
    s.store(key(1, 0), piece(7, -1, 1), true);
    CHECK(ids(s.pieces(key(1, 0))) == (Ids{{1, 5, 1}, {0, 2, 1}, {-1, 7, 1}}));
    std::map<int64_t, std::vector<Piece>> in;
    in[0] = {piece(0, 2, 3), piece(2, 0, 4)};  // the second replaces the local piece of the same map task
    in[1] = {piece(1, 1, 1), piece(4, 0, 1), piece(1, 0, 1)};
    in[2] = {};                                // a partition without rows: left as it is (absent)
    s.install("j", 1, in);
    CHECK(ids(s.pieces(key(1, 0))) == (Ids{{-1, 7, 1}, {0, 2, 4}, {1, 5, 1}, {2, 0, 3}}));
    CHECK(ids(s.pieces(key(1, 1))) == (Ids{{0, 1, 1}, {0, 4, 1}, {1, 1, 1}}));
    CHECK(s.rows(key(1, 2)) == -1);
    CHECK(s.partitions("j", 1) == 2);
  }
  {  // the empty-partition outcomes
    ShuffleStore s;
    s.replace_partition(key(1, 3), piece(-1, 0, 0));  // un-partitioned writer: a zero-row piece, 0 rows
    CHECK(s.rows(key(1, 3)) == 0 && s.pieces(key(1, 3)).size() == 1);
    s.store(key(1, 0), piece(3, 0, 0), false);  // a map task's piece without rows: no entry, -1
    CHECK(s.rows(key(1, 0)) == -1 && s.pieces(key(1, 0)).empty());
    s.store(key(1, 1), piece(3, 0, 4), false);  // ... and its retry without rows removes the earlier piece
    s.store(key(1, 1), piece(3, 0, 0), false);
    CHECK(s.rows(key(1, 1)) == -1);
    s.store(key(1, 1), piece(3, 0, 4), false);
    s.store(key(1, 1), piece(2, 0, 4), false);
    s.store(key(1, 1), piece(3, 0, 0), false);  // other tasks' pieces keep the entry
    CHECK(ids(s.pieces(key(1, 1))) == (Ids{{0, 2, 4}}));
    s.store(key(1, 2), piece(9, -1, 0), true);  // a file that holds no rows: kept, 0 rows
    CHECK(s.rows(key(1, 2)) == 0);
    s.replace_partition(key(1, 3), piece(-1, 0, 6));  // a re-run of the un-partitioned writer replaces everything
    CHECK(ids(s.pieces(key(1, 3))) == (Ids{{0, -1, 6}}));
  }
  {  // a failed task leaves nothing behind: its pieces, the un-partitioned piece of its partition; nothing else
    ShuffleStore s;
    s.store(key(1, 0), piece(2, 0, 1), false);
    s.store(key(1, 0), piece(5, 0, 1), false);
    s.store(key(1, 1), piece(2, 0, 1), false);  // the only piece there: the entry goes
    s.store(key(1, 1), piece(2, 1, 1), false);  // (another executor's task of the same id)
    s.store(key(1, 3), piece(2, 0, 1), false);
    s.replace_partition(key(2, 2), piece(-1, 0, 3));  // un-partitioned output of input partition 2, stage 2
    s.replace_partition(key(2, 5), piece(-1, 0, 3));
    s.store(key(1, 4), piece(2, 0, 1), false);
    s.store(ShuffleKey{"k", 1, 0}, piece(2, 0, 1), false);
    s.remove_task("j", 1, 2, 0);
    CHECK(ids(s.pieces(key(1, 0))) == (Ids{{0, 5, 1}}));
    CHECK(ids(s.pieces(key(1, 1))) == (Ids{{1, 2, 1}}));
    CHECK(s.rows(key(1, 3)) == -1 && s.rows(key(1, 4)) == -1);
    CHECK(s.rows(key(2, 2)) == 3 && s.rows(ShuffleKey{"k", 1, 0}) == 1);
    s.remove_task("j", 2, 2, 1);  // another executor's task: nothing of this one's
    CHECK(s.rows(key(2, 2)) == 3);
    s.remove_task("j", 2, 2, 0);
    CHECK(s.rows(key(2, 2)) == -1 && s.rows(key(2, 5)) == 3);
  }
  {  // stage and job removal; the store reports when it became empty
    ShuffleStore s;
    s.store(key(1, 0), piece(0, 0, 1), false);
    s.store(key(2, 0), piece(0, 0, 1), false);
    s.store(key(2, 1), piece(0, 0, 1), false);
    s.store(ShuffleKey{"k", 2, 0}, piece(0, 0, 1), false);
    s.remove_stage("j", 2);
    CHECK(s.rows(key(2, 0)) == -1 && s.rows(key(2, 1)) == -1 && s.rows(key(1, 0)) == 1 && s.rows(ShuffleKey{"k", 2, 0}) == 1);
    CHECK(!s.remove_job("j"));
    CHECK(s.rows(key(1, 0)) == -1 && s.rows(ShuffleKey{"k", 2, 0}) == 1);
    CHECK(s.remove_job("k"));
    CHECK(s.remove_job("k"));
    s.store(key(1, 0), piece(0, 0, 1), false);
    s.remove_all();
    CHECK(s.rows(key(1, 0)) == -1 && s.remove_job("x"));
  }
  {  // partition count: one more than the highest partition present of that job and stage
    ShuffleStore s;
    CHECK(s.partitions("j", 1) == 0);
    s.store(key(1, 4), piece(0, 0, 1), false);
    s.store(key(1, 1), piece(0, 0, 1), false);
    s.store(key(2, 9), piece(0, 0, 1), false);
    s.store(ShuffleKey{"k", 1, 7}, piece(0, 0, 1), false);
    CHECK(s.partitions("j", 1) == 5 && s.partitions("j", 2) == 10 && s.partitions("k", 1) == 8 && s.partitions("j", 3) == 0);
  }
  {  // one executor's pieces of a stage, by partition and then in reading order; the hand-over of partitions
    ShuffleStore s;
    s.store(key(1, 2), piece(0, 0, 1), false);
    s.store(key(1, 0), piece(1, 0, 2), false);
    s.store(key(1, 0), piece(1, 1, 3), false);
    s.store(key(1, 0), piece(0, 0, 4), false);
    s.store(key(1, 1), piece(-1, -1, 5), true);
    s.store(key(2, 0), piece(0, 0, 6), false);
    std::vector<StoredPiece> mine = s.of_rank("j", 1, 0);
    CHECK(mine.size() == 3);
    if (mine.size() == 3) {
      CHECK(mine[0].part == 0 && mine[0].piece.file_id == 1 && mine[0].piece.r1 == 2);
      CHECK(mine[1].part == 0 && mine[1].piece.file_id == 0 && mine[1].piece.r1 == 4);
      CHECK(mine[2].part == 2 && mine[2].piece.r1 == 1);
    }
    CHECK(s.of_rank("j", 1, -1).size() == 1 && s.of_rank("j", 3, 0).empty());
    s.remove_parts("j", 1, {0, 2, 7});
    CHECK(s.rows(key(1, 0)) == -1 && s.rows(key(1, 2)) == -1 && s.rows(key(1, 1)) == 5 && s.rows(key(2, 0)) == 6);
  }
  printf("fails=%d\n", fails);
  return fails ? 1 : 0;
}
