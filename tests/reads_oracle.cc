// reads_oracle.cc -- CPU ORACLE of the MultiPaxos read path (include/fpx.h fpx_reads_*).  TEST INFRASTRUCTURE.
//
// A naive, single-threaded restatement with the reference's own data structures: the Client's / ReadBatcher's
// per-read reply maps and the Replica's deferredReads map.  Nothing in the product links or calls this file;
// tests/reads_oracle.py compiles it into a temporary directory and binds it with ctypes.  The independent
// Python transcription it is checked against is tests/scala_transcription_reads.py.
//
// Citations: S/ = shared/src/main/scala/frankenpaxos/ in the reference tree.

#include <algorithm>
#include <climits>
#include <cstdint>
#include <map>
#include <utility>
#include <vector>

namespace fpo_reads {
// ---- MultiPaxos linearizable reads (include/fpx.h fpx_reads_*)
// Client.handleMaxSlotReply (S/multipaxos/Client.scala:851-931) / ReadBatcher.handleBatchMaxSlotReply
// (S/multipaxos/ReadBatcher.scala:568-623), with the reference's maps: states(key) = MaxSlot(id, replies)
// where replies is a map keyed by (group, acceptor), or by acceptorIndex alone for the ReadBatcher.
struct ReadTally {
  int kind, f, groups, per_group, flexible;
  struct MaxSlot { int id; std::map<std::pair<int, int>, int> replies; };
  std::map<int, MaxSlot> states;   // open reads only; a completed read leaves (PendingRead / remove)
  // 0 ok, else -5 (Grid.isReadQuorum require) with *err = reply index
  int replies(const int32_t* in, int n, int32_t* out, int* n_out, int64_t* err) {
    *n_out = 0;
    for (int i = 0; i < n; ++i) {
      const int32_t* r = in + 4 * i;
      auto it = states.find(r[0]);
      if (it == states.end() || it->second.id != r[1]) continue;   // :858-874, :572-580
      const int group = (int)((uint32_t)r[2] >> 16), acc = r[2] & 0xffff;
      const bool member = acc < per_group && (kind == 1 || group < groups);
      auto& m = it->second.replies;
      m[kind == 1 ? std::make_pair(0, acc) : std::make_pair(group, acc)] = r[3];   // :877-879, :584
      if (!member) { *err = i; return -5; }
      bool done;
      if (kind == 0 && flexible) {   // Grid.isReadQuorum: some row entirely inside
        done = false;
        for (int row = 0; row < groups && !done; ++row) {
          bool all = true;
          for (int c = 0; c < per_group; ++c) all = all && m.count({row, c});
          done = all;
        }
      } else {
        done = (int)m.size() >= f + 1;   // :880, :585
      }
      if (!done) continue;
      int mx = INT_MIN;
      for (auto& kv : m) mx = std::max(mx, kv.second);
      const int add = (kind == 0 && flexible) ? 0 : groups - 1;   // :892-898, :592-598
      int32_t* o = out + 4 * (*n_out)++;
      o[0] = r[0]; o[1] = r[1]; o[2] = (int32_t)((uint32_t)mx + (uint32_t)add); o[3] = 0;
      states.erase(it);
    }
    return 0;
  }
};

// Replica.handleDeferrableRead(s) (S/multipaxos/Replica.scala:463-529) and executeLog's deferred reads
// (:394-413): deferredReads is a map slot -> buffer of reads in arrival order.
struct DeferredReads {
  int executed_watermark = 0, capacity;
  size_t pending = 0;
  std::map<int, std::vector<int>> deferred;
  explicit DeferredReads(int cap) : capacity(cap) {}
  int request(const int32_t* in, int n, int32_t* out, int* n_out, int64_t* err) {
    *n_out = 0;
    size_t add = 0;
    for (int i = 0; i < n; ++i)
      if (in[2 * i] >= executed_watermark && pending + add++ >= (size_t)capacity) { *err = i; return -8; }
    for (int i = 0; i < n; ++i) {
      const int slot = in[2 * i], handle = in[2 * i + 1];
      if (slot >= executed_watermark) { deferred[slot].push_back(handle); ++pending; continue; }
      int32_t* o = out + 4 * (*n_out)++;
      o[0] = handle; o[1] = executed_watermark - 1; o[2] = executed_watermark - 1; o[3] = 0;   // :521-527
    }
    return 0;
  }
  int advance(int w, int32_t* out, int* n_out) {
    *n_out = 0;
    if (w < executed_watermark) return -1;
    while (!deferred.empty() && deferred.begin()->first < w) {
      const int slot = deferred.begin()->first;
      for (int h : deferred.begin()->second) {
        int32_t* o = out + 4 * (*n_out)++;
        o[0] = h; o[1] = slot - 1; o[2] = slot; o[3] = 0;   // processDeferredReads before executedWatermark += 1
        --pending;
      }
      deferred.erase(deferred.begin());
    }
    executed_watermark = w;
    return 0;
  }
};

}  // namespace fpo_reads

using namespace fpo_reads;

extern "C" {

void* fpo_rt_new(int kind, int f, int groups, int per_group, int flexible) {
  return new ReadTally{kind, f, groups, per_group, flexible, {}};
}
void fpo_rt_free(void* p) { delete (ReadTally*)p; }
void fpo_rt_open(void* p, const int32_t* in, int n) {
  for (int i = 0; i < n; ++i) ((ReadTally*)p)->states[in[2 * i]] = ReadTally::MaxSlot{in[2 * i + 1], {}};
}
int fpo_rt_replies(void* p, const int32_t* in, int n, int32_t* out, int* n_out, int64_t* err) {
  *err = -1;
  return ((ReadTally*)p)->replies(in, n, out, n_out, err);
}
void* fpo_dr_new(int capacity) { return new DeferredReads(capacity); }
void fpo_dr_free(void* p) { delete (DeferredReads*)p; }
int fpo_dr_request(void* p, const int32_t* in, int n, int32_t* out, int* n_out, int64_t* err) {
  *err = -1;
  return ((DeferredReads*)p)->request(in, n, out, n_out, err);
}
int fpo_dr_advance(void* p, int w, int32_t* out, int* n_out) { return ((DeferredReads*)p)->advance(w, out, n_out); }
int fpo_dr_pending(void* p) { return (int)((DeferredReads*)p)->pending; }

}  // extern "C"
