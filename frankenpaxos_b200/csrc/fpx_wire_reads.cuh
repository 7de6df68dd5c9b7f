// fpx_wire_reads.cuh -- wire codec of the MultiPaxos replica and read path (S/multipaxos/MultiPaxos.proto):
//   replica decode   ReplicaInbound :563-576 -> fpx_chosen records (Chosen) and fpx_read_request records (one per
//                    Command of the six read members), count -> tile offsets -> emit, cut at the order split;
//   reads decode     ClientInbound :489-500 / ReadBatcherInbound :513-523 -> one fpx_max_slot_reply per message;
//   encoders         the acceptor's MaxSlotReply / BatchMaxSlotReply and the ReadRequest / ReadRequestBatch of a
//                    completed read, size -> tile offsets -> emit with the gathered bytes copied by the CTA's warps.
// Parsing rules as in fpx_wire.cuh; nested messages that are parsed (a member given again, Command, CommandId) are
// merged as protobuf-java's mergeFrom builds them and `required` is checked on the merged result at every level.
#pragma once
#include "fpx_reads.cuh"
#include "fpx_wire.cuh"

namespace fpx {

// The member that stands once the whole message is read (the last one on the wire) and the position of the first
// occurrence of its final run: protobuf-java merges a member given again and drops it when another member follows.
// Field numbers 1..members with wire type 2 are members; anything else is skipped as unknown.
template <bool kS>
__device__ __forceinline__ bool wire_oneof_run(WireReader<kS> r, int members, int* which, uint32_t* run, uint32_t* blo,
                                               uint32_t* bhi) {
  *which = 0; *run = r.p; *blo = *bhi = 0;
  while (!r.done()) {
    const uint32_t tpos = r.p;
    const uint32_t tag = r.tag();
    if (!r.ok) return false;
    const int wt = (int)(tag & 7);
    if (wt == 2) {
      const uint32_t n = r.small();
      if (!r.ok || r.end - r.p < n) return false;
      const int f = (int)(tag >> 3);
      if (f <= members) {
        if (f != *which) { *which = f; *run = tpos; }
        *blo = r.p; *bhi = r.p + n;
      }
      r.p += n;
    } else if (!r.skip(wt)) {
      return false;
    }
  }
  return true;
}

// CommandId {client_address = 1, client_pseudonym = 2, client_id = 3} (MultiPaxos.proto:188-196), merged: have-bits
// accumulate in *have (bit f - 1), a later value wins.  *aoff / *alen: the last client_address's bytes.
template <bool kS>
__device__ __forceinline__ bool wire_command_id(WireReader<kS> b, unsigned* have, int* pseudo, int* id, uint32_t* aoff,
                                                uint32_t* alen) {
  while (!b.done()) {
    const uint32_t tag = b.tag();
    if (!b.ok) return false;
    const int f = (int)(tag >> 3), wt = (int)(tag & 7);
    if (f == 1 && wt == 2) {
      const uint32_t n = b.small();
      if (!b.ok || b.end - b.p < n) return false;
      *aoff = b.p; *alen = n; b.p += n;
      *have |= 1u;
    } else if ((f == 2 || f == 3) && wt == 0) {
      const int v = (int)b.int32();
      if (!b.ok) return false;
      if (f == 2) *pseudo = v; else *id = v;
      *have |= 1u << (f - 1);
    } else if (!b.skip(wt)) {
      return false;
    }
  }
  return true;
}

// Command {command_id = 1, command = 2} (:198-204), both required, CommandId's three fields too
template <bool kS>
__device__ __forceinline__ bool wire_command(WireReader<kS> b) {
  unsigned have = 0, cid = 0;
  int pseudo = 0, id = 0;
  uint32_t aoff = 0, alen = 0;
  while (!b.done()) {
    const uint32_t tag = b.tag();
    if (!b.ok) return false;
    const int f = (int)(tag >> 3), wt = (int)(tag & 7);
    if ((f == 1 || f == 2) && wt == 2) {
      const uint32_t n = b.small();
      if (!b.ok || b.end - b.p < n) return false;
      if (f == 1) {
        WireReader<kS> s = b;
        s.end = b.p + n;
        if (!wire_command_id(s, &cid, &pseudo, &id, &aoff, &alen)) return false;
      }
      have |= 1u << (f - 1);
      b.p += n;
    } else if (!b.skip(wt)) {
      return false;
    }
  }
  return have == 3u && cid == 7u;
}

// ---------------------------------------------------------------------------
// ReplicaInbound {chosen = 1, read_request = 2, sequential_read_request = 3, eventual_read_request = 4,
// read_request_batch = 5, sequential_read_request_batch = 6, eventual_read_request_batch = 7}
// ---------------------------------------------------------------------------
constexpr int kRwThreads = kWireDecThreads;   // messages per tile of the replica decode

// field number of a read member's Command(s); its slot is field 1 where it has one
__host__ __device__ constexpr int rw_command_field(int which) { return which == 4 || which == 7 ? 1 : 2; }
__host__ __device__ constexpr bool rw_singular(int which) { return which >= 2 && which <= 4; }

struct RwMsg {
  int slot, cnt;              // reads: the Commands of the run
  unsigned have;              // bit 0: slot, bit 1: the value (Chosen) / a Command
  uint32_t voff, vlen;        // Chosen: the CommandBatchOrNoop (reader positions)
};
// where an emitting parse writes the run's read records
struct RwEmit {
  fpx_read_request* reads;
  int2* spans;
  long long at;               // output index of the run's first Command
  int limit;                  // the Commands the count pass found: no record is written past them
  int slot, handle_base;
  uint32_t base;              // reader position -> buffer offset
};

// The final run of member `which` from reader position `run` on, merged into m.  kEmit: one read record per Command.
template <bool kEmit, bool kS>
__device__ __forceinline__ bool rw_run(WireReader<kS> r, uint32_t run, int which, RwMsg& m, const RwEmit* o) {
  r.p = run;
  const int cf = rw_command_field(which);
  const bool has_slot = which != 4 && which != 7;
  while (!r.done()) {
    const uint32_t tag = r.tag();
    if (!r.ok) return false;
    const int wt = (int)(tag & 7);
    if (wt != 2 || (int)(tag >> 3) != which) {   // an unknown field (the run holds no other member)
      if (!r.skip(wt)) return false;
      continue;
    }
    const uint32_t len = r.small();
    if (!r.ok || r.end - r.p < len) return false;
    WireReader<kS> b = r;
    b.end = r.p + len;
    r.p += len;
    while (!b.done()) {
      const uint32_t tag2 = b.tag();
      if (!b.ok) return false;
      const int f = (int)(tag2 >> 3), wt2 = (int)(tag2 & 7);
      if (f == 1 && wt2 == 0 && (which == 1 || has_slot)) {
        m.slot = (int)b.int32();
        if (!b.ok) return false;
        m.have |= 1u;
      } else if (which == 1 && f == 2 && wt2 == 2) {          // Chosen.command_batch_or_noop: located, not parsed
        const uint32_t n = b.small();
        if (!b.ok || b.end - b.p < n || (m.have & 2u)) return false;   // a second one would merge: unsupported
        m.voff = b.p; m.vlen = n; b.p += n;
        m.have |= 2u;
      } else if (which != 1 && f == cf && wt2 == 2) {
        const uint32_t n = b.small();
        if (!b.ok || b.end - b.p < n) return false;
        if (rw_singular(which) && (m.have & 2u)) return false;      // a second Command would merge: unsupported
        WireReader<kS> s = b;
        s.end = b.p + n;
        if (!wire_command(s)) return false;
        if (kEmit && m.cnt < o->limit) {
          const long long k = o->at + m.cnt;
          o->reads[k] = fpx_read_request{o->slot, (int32_t)((uint32_t)o->handle_base + (uint32_t)k)};
          o->spans[k] = make_int2((int)(b.p + o->base), (int)n);
        }
        ++m.cnt;
        m.have |= 2u;
        b.p += n;
      } else if (!b.skip(wt2)) {
        return false;
      }
    }
  }
  // "Message missing required fields"
  if (which == 1 || which == 2 || which == 3) return m.have == 3u;
  if (which == 4) return (m.have & 2u) != 0;
  if (which == 5 || which == 6) return (m.have & 1u) != 0;
  return true;
}

struct RwDecodeParams {
  const uint8_t* bytes;       // 16-byte aligned
  const int32_t* offs;        // n + 1
  int32_t n;
  int32_t value_id_base, handle_base, reads_cap;
  int32_t* kind;
  fpx_chosen* chosen;         // dense, capacity n
  int2* chosen_spans;
  fpx_read_request* reads;    // dense, capacity reads_cap
  int2* read_spans;
  int32_t* counts;            // {n_chosen, n_reads, split}
  // scratch
  int32_t* cnt;               // [n] Commands of a read message
  int32_t* slot;              // [n]
  int2* vspan;                // [n] a Chosen's value span (buffer offsets)
  uint32_t* tile_reads;       // [tiles + 1] Commands per tile, then exclusive offsets
  uint32_t* tile_chosen;      // [tiles + 1] Chosen messages per tile, then exclusive offsets
  int32_t* first_chosen;      // [tiles] first Chosen of the tile (INT_MAX: none)
  int32_t* first_read;        // [tiles] first read message of the tile
  int32_t* read_after;        // [tiles] first read message of the tile after the tile's first Chosen
  DevStatus* st;
};

__device__ __forceinline__ bool rw_is_read(int kind) { return kind >= 2 && kind <= 7; }

// pass 1: parse every message, its kind, Command count, slot and value span; per-tile counts and the order summary
__global__ void __launch_bounds__(kRwThreads) rw_count_kernel(RwDecodeParams P) {
  __shared__ __align__(16) uint8_t s_buf[kWireStage + 32];
  __shared__ int s_first_chosen, s_first_read, s_read_after;
  if (threadIdx.x == 0) { s_first_chosen = INT_MAX; s_first_read = INT_MAX; s_read_after = INT_MAX; }
  const int m0 = blockIdx.x * kRwThreads;
  const int m1 = min(P.n, m0 + kRwThreads);
  const WireSpan w = wire_stage_span(P.bytes, P.offs, P.n, m0, m1, s_buf);   // its barrier publishes the inits
  const int i = m0 + threadIdx.x;
  int kind = 0;
  RwMsg m{-1, 0, 0u, 0u, 0u};
  if (i < m1) {
    bool ok = false;
    wire_read(w, s_buf, P.bytes, P.offs[i], P.offs[i + 1], [&](auto r, uint32_t rebase) {
      uint32_t run = 0, blo, bhi;
      ok = wire_oneof_run(r, 7, &kind, &run, &blo, &bhi) && (kind == 0 || rw_run<false>(r, run, kind, m, nullptr));
      m.voff += rebase;
    });
    if (!ok) {
      report_error(P.st, FPX_ERR_WIRE, i);
      kind = 0;
    }
    P.kind[i] = kind;
    P.cnt[i] = rw_is_read(kind) ? m.cnt : 0;
    P.slot[i] = kind == 4 || kind == 7 ? -1 : m.slot;            // the eventual reads' slot (fpx_reads_replica)
    P.vspan[i] = kind == 1 ? make_int2((int)m.voff, (int)m.vlen) : make_int2(0, 0);
    if (kind == 1) atomicMin(&s_first_chosen, i);
    if (rw_is_read(kind)) atomicMin(&s_first_read, i);
  }
  const uint32_t reads = cta_reduce<kRwThreads>((uint32_t)(rw_is_read(kind) ? m.cnt : 0), ScanSum());
  const uint32_t chosen = cta_reduce<kRwThreads>((uint32_t)(kind == 1), ScanSum());   // its barriers publish the mins
  if (rw_is_read(kind) && i > s_first_chosen) atomicMin(&s_read_after, i);
  __syncthreads();
  if (threadIdx.x == 0) {
    P.tile_reads[blockIdx.x] = reads;
    P.tile_chosen[blockIdx.x] = chosen;
    P.first_chosen[blockIdx.x] = s_first_chosen;
    P.first_read[blockIdx.x] = s_first_read;
    P.read_after[blockIdx.x] = s_read_after;
  }
}

// one CTA: split = the first read message after the batch's first Chosen (n if none)
__global__ void __launch_bounds__(1024) rw_split_kernel(RwDecodeParams P, int tiles) {
  __shared__ int s_c0, s_split;
  if (threadIdx.x == 0) { s_c0 = INT_MAX; s_split = INT_MAX; }
  __syncthreads();
  for (int t = threadIdx.x; t < tiles; t += 1024) atomicMin(&s_c0, P.first_chosen[t]);
  __syncthreads();
  const int c0 = s_c0;
  if (c0 != INT_MAX) {
    const int t0 = c0 / kRwThreads;
    for (int t = t0 + threadIdx.x; t < tiles; t += 1024) atomicMin(&s_split, t == t0 ? P.read_after[t] : P.first_read[t]);
  }
  __syncthreads();
  if (threadIdx.x == 0) P.counts[2] = s_split == INT_MAX ? P.n : s_split;
}

// pass 2 (after the tile offsets and the split): the records of messages [0, split)
__global__ void __launch_bounds__(kRwThreads) rw_emit_kernel(RwDecodeParams P) {
  const int split = __ldcg(&P.counts[2]);
  const int m0 = blockIdx.x * kRwThreads;
  if (m0 > split) return;
  const int m1 = min(P.n, m0 + kRwThreads);
  __shared__ __align__(16) uint8_t s_buf[kWireStage + 32];
  // the count pass's window, so that a message is read from the same bytes (and the same kind of reader) it was
  // checked in: a message it accepted lies inside [w.lo, w.hi) whatever the offsets of the others
  const WireSpan w = wire_stage_span(P.bytes, P.offs, P.n, m0, m1, s_buf);
  const int i = m0 + threadIdx.x;
  const bool mine = i < m1 && i < split;
  const int kind = mine ? __ldcg(&P.kind[i]) : 0;
  const int cnt = mine ? __ldcg(&P.cnt[i]) : 0;
  const uint32_t base_r = __ldcg(&P.tile_reads[blockIdx.x]), base_c = __ldcg(&P.tile_chosen[blockIdx.x]);
  uint32_t tot_r, tot_c;
  const uint32_t off_r = base_r + cta_scan<kRwThreads, true>((uint32_t)cnt, ScanSum(), &tot_r);
  const uint32_t off_c = base_c + cta_scan<kRwThreads, true>((uint32_t)(kind == 1), ScanSum(), &tot_c);
  // the counts over [0, split): the exclusive offsets at `split`, or the totals of the last tile when split = n
  if (split < m1 && i == split) {
    P.counts[0] = (int32_t)off_c; P.counts[1] = (int32_t)off_r;
  } else if (split == m1 && m1 == P.n && threadIdx.x == 0) {
    P.counts[0] = (int32_t)(base_c + tot_c); P.counts[1] = (int32_t)(base_r + tot_r);
  }
  if (!mine) return;
  if (kind == 1) {
    P.chosen[off_c] = fpx_chosen{__ldcg(&P.slot[i]), (int32_t)((uint32_t)P.value_id_base + (uint32_t)i)};
    P.chosen_spans[off_c] = __ldcg(&P.vspan[i]);
    return;
  }
  if (!rw_is_read(kind) || cnt == 0) return;
  if ((long long)off_r + cnt > (long long)P.reads_cap) {
    report_error(P.st, FPX_ERR_OVERFLOW_FULL, i);
    return;
  }
  // a message outside the span: the count pass refused it already
  wire_read(w, s_buf, P.bytes, P.offs[i], P.offs[i + 1], [&](auto r, uint32_t rebase) {
    RwMsg m{-1, 0, 0u, 0u, 0u};
    int which;
    uint32_t run, blo, bhi;
    const RwEmit o{P.reads, P.read_spans, (long long)off_r, cnt, __ldcg(&P.slot[i]), P.handle_base, rebase};
    if (wire_oneof_run(r, 7, &which, &run, &blo, &bhi)) rw_run<true>(r, run, which, m, &o);
  });
}

// ---------------------------------------------------------------------------
// ClientInbound {.., max_slot_reply = 4, read_reply = 5} / ReadBatcherInbound {.., batch_max_slot_reply = 4}
// ---------------------------------------------------------------------------
struct RdDecodeParams {
  const uint8_t* bytes;       // 16-byte aligned
  const int32_t* offs;        // n + 1
  int32_t n;
  int32_t batcher;            // FPX_READS_READ_BATCHER
  int32_t key_cap;
  int32_t* kind;
  int4* out;                  // fpx_max_slot_reply
  int2* spans;
  unsigned long long* err_word;
};

// the run of member 4 merged: MaxSlotReply {command_id, group_index, acceptor_index, slot} (:323-331) or
// BatchMaxSlotReply {read_batcher_index, read_batcher_id, acceptor_index, slot} (:341-349), all required
template <bool kS>
__device__ __forceinline__ bool rd_reply_run(WireReader<kS> r, uint32_t run, bool batcher, int v[4], int* pseudo, int* id) {
  r.p = run;
  unsigned have = 0, cid = 0;
  uint32_t aoff = 0, alen = 0;
  while (!r.done()) {
    const uint32_t tag = r.tag();
    if (!r.ok) return false;
    const int wt = (int)(tag & 7);
    if (wt != 2 || (tag >> 3) != 4u) {
      if (!r.skip(wt)) return false;
      continue;
    }
    const uint32_t len = r.small();
    if (!r.ok || r.end - r.p < len) return false;
    WireReader<kS> b = r;
    b.end = r.p + len;
    r.p += len;
    while (!b.done()) {
      const uint32_t tag2 = b.tag();
      if (!b.ok) return false;
      const int f = (int)(tag2 >> 3), wt2 = (int)(tag2 & 7);
      if (!batcher && f == 1 && wt2 == 2) {
        const uint32_t n = b.small();
        if (!b.ok || b.end - b.p < n) return false;
        WireReader<kS> s = b;
        s.end = b.p + n;
        if (!wire_command_id(s, &cid, pseudo, id, &aoff, &alen)) return false;
        have |= 1u;
        b.p += n;
      } else if (f >= (batcher ? 1 : 2) && f <= 4 && wt2 == 0) {
        const int x = (int)b.int32();
        if (!b.ok) return false;
        if (f == 1) v[0] = x; else if (f == 2) v[1] = x; else if (f == 3) v[2] = x; else v[3] = x;
        have |= 1u << (f - 1);
      } else if (!b.skip(wt2)) {
        return false;
      }
    }
  }
  return have == 0xfu && (batcher || cid == 7u);
}

__global__ void __launch_bounds__(kWireDecThreads) rd_wire_decode_kernel(RdDecodeParams P) {
  __shared__ __align__(16) uint8_t s_buf[kWireStage + 32];
  const int m0 = blockIdx.x * kWireDecThreads;
  const int m1 = min(P.n, m0 + kWireDecThreads);
  const WireSpan w = wire_stage_span(P.bytes, P.offs, P.n, m0, m1, s_buf);
  const int i = m0 + threadIdx.x;
  if (i >= m1) return;
  const bool batcher = P.batcher != 0;
  int which = 0, pseudo = 0, id = 0;
  int v[4] = {0, 0, 0, 0};
  uint32_t blo = 0, bhi = 0, rebase = 0;
  bool ok = false;
  wire_read(w, s_buf, P.bytes, P.offs[i], P.offs[i + 1], [&](auto r, uint32_t base) {
    uint32_t run = 0;
    ok = wire_oneof_run(r, batcher ? 4 : 5, &which, &run, &blo, &bhi) &&
         (which != 4 || rd_reply_run(r, run, batcher, v, &pseudo, &id));
    rebase = base;
  });
  int4 rec = make_int4(-1, 0, 0, 0);
  if (!ok) {
    report_error(P.err_word, FPX_ERR_WIRE, i);
    which = 0;
  } else if (which == 4) {
    // voter = group << 16 | acceptor; a field outside [0, 2^15) names no voter (-1: the tally's BAD_ACCEPTOR rule)
    const int g = batcher ? 0 : v[1], acc = v[2];
    const int voter = (uint32_t)g < 0x8000u && (uint32_t)acc < 0x8000u ? (g << 16 | acc) : -1;
    if (batcher) {
      const int key = v[1] % P.key_cap;                             // floorMod(read_batcher_id, key_capacity)
      rec = make_int4(key < 0 ? key + P.key_cap : key, v[1], voter, v[3]);
    } else {
      rec = make_int4(pseudo, id, voter, v[3]);
    }
  }
  P.kind[i] = which;
  P.out[i] = rec;
  P.spans[i] = which ? make_int2((int)(blo + rebase), (int)(bhi - blo)) : make_int2(0, 0);
}

// ---------------------------------------------------------------------------
// encoders: the acceptor's MaxSlotReply / BatchMaxSlotReply, and a completed read's ReadRequest / ReadRequestBatch
// ---------------------------------------------------------------------------
struct RdEncodeParams {
  WireEnc enc;                // enc.src: the request batch (client_address) or the arena
  int32_t read_requests;      // 0: max-slot replies (kind[] + fpx_wire_rec), 1: read requests (fpx_read_slot)
  int32_t outer;              // read requests: the member's tag byte (0x12 read_request, 0x2a read_request_batch)
  const int32_t* kind;
  const int4* in;
  int32_t src_len;            // max-slot replies: bytes in the request batch
  const int32_t* value_offs;  // read requests
  int32_t num_values;
  int32_t groups, per_group;  // max-slot replies: the voters of the config
};

// One message: outer tag, [CommandId{client_address = gathered, pseudo, id} as field 1], int32 fields
// f1 .. f1 + nf - 1, [the gathered bytes as the body's tail]
struct RdMsg {
  int outer;                  // 0: a zero-length message
  bool cid;
  int f1, nf;
  int v[4];
  int pseudo, id;
  int src, glen;
};

__device__ __forceinline__ RdMsg rd_enc_msg(const RdEncodeParams& P, int i, int* code) {
  RdMsg m{};
  const int4 r = P.in[i];
  if (P.read_requests) {                       // {slot, command*}: arena entry key = the command field(s)
    m.outer = P.outer; m.f1 = 1; m.nf = 1; m.v[0] = r.z;
    const int key = r.x;
    long long len = -1;
    if ((uint32_t)key < (uint32_t)P.num_values) { m.src = P.value_offs[key]; len = (long long)P.value_offs[key + 1] - m.src; }
    if (len < 0) { *code = FPX_ERR_INVALID_ARG; m.outer = 0; return m; }
    m.glen = (int)len;
    return m;
  }
  const int kind = P.kind[i];
  if (kind != 3 && kind != 4) return m;
  // the request's body: {0, 0, body_off, body_len} as fpx_wire_decode_inbound writes it
  WireReader<false> b{0u, P.enc.src, (uint32_t)r.z, (uint32_t)r.z + (uint32_t)r.w, true};
  bool ok = r.z >= 0 && r.w >= 0 && (long long)r.z + r.w <= P.src_len;
  unsigned have = 0, cid = 0;
  uint32_t aoff = 0, alen = 0;
  int x[2] = {0, 0};
  while (ok && !b.done()) {
    const uint32_t tag = b.tag();
    if (!b.ok) { ok = false; break; }
    const int f = (int)(tag >> 3), wt = (int)(tag & 7);
    if (kind == 3 && f == 1 && wt == 2) {      // MaxSlotRequest {command_id} (:316-321), merged
      const uint32_t n = b.small();
      if (!b.ok || b.end - b.p < n) { ok = false; break; }
      WireReader<false> s = b;
      s.end = b.p + n;
      if (!wire_command_id(s, &cid, &m.pseudo, &m.id, &aoff, &alen)) { ok = false; break; }
      have |= 1u;
      b.p += n;
    } else if (kind == 4 && (f == 1 || f == 2) && wt == 0) {   // BatchMaxSlotRequest {index, id} (:333-339)
      const int v = (int)b.int32();
      if (!b.ok) { ok = false; break; }
      if (f == 1) x[0] = v; else x[1] = v;
      have |= 1u << (f - 1);
    } else if (!b.skip(wt)) {
      ok = false;
    }
  }
  if (!ok || (kind == 3 ? have != 1u || cid != 7u : have != 3u)) { *code = FPX_ERR_WIRE; return m; }
  const int g = r.x >> 16, acc = r.x & 0xffff;
  if (r.x < 0 || g >= P.groups || acc >= P.per_group) { *code = FPX_ERR_INVALID_ARG; return m; }
  m.outer = 0x22;                              // ClientInbound.max_slot_reply = ReadBatcherInbound.batch_max_slot_reply = 4
  if (kind == 3) {                             // MaxSlotReply {command_id, group_index, acceptor_index, slot}
    m.cid = true; m.src = (int)aoff; m.glen = (int)alen;
    m.f1 = 2; m.nf = 3; m.v[0] = g; m.v[1] = acc; m.v[2] = r.y;
  } else {                                     // BatchMaxSlotReply {read_batcher_index, read_batcher_id, acceptor, slot}
    m.f1 = 1; m.nf = 4; m.v[0] = x[0]; m.v[1] = x[1]; m.v[2] = acc; m.v[3] = r.y;
  }
  return m;
}

__device__ __forceinline__ int rd_cid_body(const RdMsg& m) {
  return 1 + wire_varint_size((unsigned long long)m.glen) + m.glen + 2 + wire_int32_size(m.pseudo) + wire_int32_size(m.id);
}
__device__ __forceinline__ int rd_msg_body(const RdMsg& m) {
  int b = 0;
  if (m.cid) { const int c = rd_cid_body(m); b += 1 + wire_varint_size((unsigned long long)c) + c; }
#pragma unroll
  for (int k = 0; k < 4; ++k)
    if (k < m.nf) b += 1 + wire_int32_size(m.v[k]);
  if (!m.cid) b += m.glen;
  return b;
}
__device__ __forceinline__ int rd_msg_size(const RdMsg& m) {
  if (!m.outer) return 0;
  const int b = rd_msg_body(m);
  return 1 + wire_varint_size((unsigned long long)b) + b;
}

struct RdWireCodec {
  using Params = RdEncodeParams;
  using Msg = RdMsg;
  static __device__ __forceinline__ bool stand_down(const Params&) { return false; }
  static __device__ __forceinline__ Msg msg(const Params& P, int i, int* code) { return rd_enc_msg(P, i, code); }
  static __device__ __forceinline__ int size(const Params&, const Msg& m) { return rd_msg_size(m); }
  static __device__ __forceinline__ int size_of(const Params& P, int i, int* code) { return rd_msg_size(rd_enc_msg(P, i, code)); }
  // the client_address inside the CommandId, else the arena's bytes as the body's tail
  static __device__ __forceinline__ uint8_t* head(const Params&, const Msg& m, uint8_t* p, int* gsrc, int* glen) {
    *p++ = (uint8_t)m.outer;
    p = wire_put_varint(p, (unsigned long long)rd_msg_body(m));
    uint8_t* gdst = nullptr;
    if (m.cid) {
      *p++ = 0x0a; p = wire_put_varint(p, (unsigned long long)rd_cid_body(m));
      *p++ = 0x0a; p = wire_put_varint(p, (unsigned long long)m.glen);
      gdst = p; p += m.glen;
      p = wire_put_int32(p, 2, m.pseudo); p = wire_put_int32(p, 3, m.id);
    }
#pragma unroll
    for (int k = 0; k < 4; ++k)
      if (k < m.nf) p = wire_put_int32(p, m.f1 + k, m.v[k]);
    if (!m.cid) gdst = p;
    *gsrc = m.src; *glen = m.glen;
    return gdst;
  }
};

}  // namespace fpx
