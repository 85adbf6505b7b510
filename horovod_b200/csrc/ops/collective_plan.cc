#include "collective_plan.h"
#include <algorithm>
#include <string>
#include "gpu_ops.h"

namespace hvd {

namespace {
int64_t Align16(int64_t b) { return (b + 15) / 16 * 16; }
int64_t Align128(int64_t b) { return (b + 127) / 128 * 128; }

// `grid_bytes` sizes the grid and MUST be the same number on every rank (CTA b rendezvouses with CTA b of its peers): a
// 4-byte broadcast is one CTA and one flag per peer, not comm_ctas of them.
void AddExchange(Plan* plan, std::vector<kern::CopyDesc>& sends, std::vector<kern::CopyDesc>& recvs, int max_ctas,
                 int64_t grid_bytes) {
  PlanLaunch l;
  l.sends.swap(sends);
  l.recvs.swap(recvs);
  l.ctas = (int)std::max<int64_t>(1, std::min<int64_t>(max_ctas, (grid_bytes + 32767) / 32768));
  plan->push_back(std::move(l));
}

std::string Str(int64_t v) { return std::to_string(v); }
}  // namespace

// Small messages are latency bound (few CTAs = cheap flag barrier, SMs left to compute); >= 64 MiB of plain tensors are
// bound by the local pack / unpack phases, which need two CTAs per SM (ncu: 12.5 % warps active at one).
int CtasFor(int variant, int64_t seg_bytes, int n, int comm_ctas, int64_t large_msg_ctas) {
  const int64_t per = variant == kern::kOneShot ? 8192 : (int64_t)4096 * n;  // >= 2 rows (one-shot) or one row per rank (two-shot) per CTA
  // (a one-shot CTA makes four dependent NVLink trips, so a 1 MiB message wants more than 16 CTAs)
  const int64_t cap_ctas = seg_bytes <= (256 << 10) ? std::min<int64_t>(comm_ctas, 16)
                         : seg_bytes <= (16 << 20) ? std::min<int64_t>(comm_ctas, 64)
                         : seg_bytes < (64 << 20) ? comm_ctas : std::max<int64_t>(comm_ctas, large_msg_ctas);
  return (int)std::max<int64_t>(1, std::min<int64_t>(cap_ctas, (seg_bytes + per - 1) / per));
}

// Every rank packs the same pieces at the same offsets and reduces the whole segment, so the plan is the same on every
// rank up to the tensor addresses.  A piece that does not fit the rest of the segment is split across segments.
Status PlanAllreduce(int n, const std::vector<PlanTensor>& ts, const ReduceParams& rp, DataType wire, const AllreducePolicy& pol,
                     int64_t cap, int comm_ctas, Plan* plan) {
  cap = cap / 128 * 128;
  if (cap < 128) return Status::InvalidArgument("allreduce: a symmetric buffer of " + Str(cap) + " bytes cannot hold 128 bytes");
  const int64_t esz = (int64_t)DataTypeSize(rp.dtype), wsz = (int64_t)DataTypeSize(wire);
  const bool multimem = pol.multicast && MultimemReduces(wire, rp.op);
  PlanLaunch l;  // the segment being filled
  int64_t seg_bytes = 0;
  auto flush = [&]() {
    if (l.table.empty()) return;
    kern::AllreduceArgs& a = l.args;
    a.ndesc = (int)l.table.size();
    a.total_bytes = seg_bytes;
    a.reduce_lo = 0; a.reduce_hi = seg_bytes;
    a.prescale = rp.prescale; a.postscale = rp.postscale;
    a.op = (int)rp.op; a.dtype = (int)rp.dtype; a.wire_dtype = (int)wire;
    if (pol.variant == "oneshot") a.variant = kern::kOneShot;
    else if (pol.variant == "twoshot") a.variant = kern::kTwoShot;
    else if (pol.variant == "nvls" && multimem) a.variant = kern::kNvls;
    else if (seg_bytes <= pol.oneshot_max_bytes) a.variant = kern::kOneShot;
    // in-switch reduction pays off from 4 GPUs (measured: slower than two-shot at N=2)
    else if (multimem && n >= 4 && seg_bytes >= pol.nvls_min_bytes) a.variant = kern::kNvls;
    else a.variant = kern::kTwoShot;
    l.reduce = true;
    l.ctas = CtasFor(a.variant, seg_bytes, n, comm_ctas, pol.large_msg_ctas);
    plan->push_back(std::move(l));
    l = PlanLaunch();
    seg_bytes = 0;
  };
  for (const PlanTensor& t : ts) {
    const int64_t count = t.dims[0];
    for (int64_t done = 0; done < count;) {
      if (cap - seg_bytes < 128) flush();
      const int64_t take = std::min(count - done, (cap - seg_bytes) / wsz);
      l.table.push_back({(const char*)t.in + done * esz, (char*)t.out + done * esz, seg_bytes, take});
      seg_bytes += Align128(take * wsz);
      done += take;
    }
  }
  flush();
  return Status::OK();
}

// The fused buffer is laid out destination-rank major — region q holds block q of EVERY tensor of the (fused) response —
// so each rank reduces one contiguous range straight into its output tensors: one launch per segment that fits the
// buffer.  A tensor whose blocks do not fit is split into element windows [w0, w0 + len) of every block.
Status PlanReducescatter(int me, int n, const std::vector<PlanTensor>& ts, const ReduceParams& rp, int64_t cap, int comm_ctas,
                         Plan* plan) {
  const int64_t esz = (int64_t)DataTypeSize(rp.dtype);
  const int64_t region_cap = cap / n / 128 * 128;  // bytes available to one destination region
  if (region_cap < 128)
    return Status::InvalidArgument("reducescatter: a symmetric buffer of " + Str(cap) + " bytes has no 128-byte region for each of " +
                                   Str(n) + " ranks");
  struct Item { const PlanTensor* t; std::vector<int64_t> cnt, boff; };  // per-destination block: elements, element offset
  std::vector<Item> items(ts.size());
  for (size_t ti = 0; ti < ts.size(); ++ti) {
    std::vector<int64_t> rows;
    ReducescatterRows(ts[ti].dims[0], n, &rows);
    Item& it = items[ti];
    it.t = &ts[ti]; it.cnt.assign(n, 0); it.boff.assign(n + 1, 0);
    for (int i = 0; i < n; ++i) { it.cnt[i] = rows[i] * ts[ti].row; it.boff[i + 1] = it.boff[i] + it.cnt[i]; }
  }
  // one launch over pieces {tensor, element window [w0, w0 + len) inside every destination block}
  struct Piece { const Item* it; int64_t w0, len; };
  std::vector<Piece> seg;
  std::vector<int64_t> used(n, 0);  // bytes used in region q by the current segment
  auto flush = [&]() {
    if (seg.empty()) return;
    const int64_t W = Align128(*std::max_element(used.begin(), used.end()));
    PlanLaunch l;
    l.reduce = true;
    std::vector<kern::TensorDesc>& table = l.table;
    table.reserve(seg.size() * (n + 1));
    for (int q = 0; q < n; ++q) {
      int64_t off = (int64_t)q * W;
      for (auto& pc : seg) {
        const int64_t c = std::max<int64_t>(0, std::min(pc.len, pc.it->cnt[q] - pc.w0));
        kern::TensorDesc d;
        d.in = (const char*)pc.it->t->in + (pc.it->boff[q] + pc.w0) * esz; d.out = nullptr; d.offset = off; d.count = c;
        table.push_back(d);
        off += Align128(c * esz);
      }
    }
    const int nin = (int)table.size();
    int64_t off = (int64_t)me * W;
    for (auto& pc : seg) {
      const int64_t c = std::max<int64_t>(0, std::min(pc.len, pc.it->cnt[me] - pc.w0));
      kern::TensorDesc d;
      d.in = nullptr; d.out = (char*)pc.it->t->out + pc.w0 * esz; d.offset = off; d.count = c;
      table.push_back(d);
      off += Align128(c * esz);
    }
    kern::AllreduceArgs& a = l.args;
    a.ndesc = nin;
    a.nout = (int)seg.size();
    a.total_bytes = (int64_t)n * W;
    a.reduce_lo = (int64_t)me * W; a.reduce_hi = off;
    a.prescale = rp.prescale; a.postscale = rp.postscale;
    a.op = (int)rp.op; a.dtype = (int)rp.dtype; a.wire_dtype = (int)rp.dtype;
    a.variant = kern::kOneShot;
    a.oneshot_nvls = (rp.nvls && a.total_bytes >= rp.nvls_min_bytes) ? 1 : 0;
    l.ctas = (int)std::max<int64_t>(1, std::min<int64_t>(comm_ctas, (a.total_bytes + 16383) / 16384));
    plan->push_back(std::move(l));
    seg.clear(); used.assign(n, 0);
  };
  for (auto& it : items) {
    const int64_t maxcnt = *std::max_element(it.cnt.begin(), it.cnt.end());
    int64_t w0 = 0;
    while (w0 < maxcnt) {
      int64_t room = region_cap - *std::max_element(used.begin(), used.end());
      if (room < 128) { flush(); room = region_cap; }
      const int64_t len = std::min(maxcnt - w0, room / esz);
      seg.push_back({&it, w0, len});
      for (int q = 0; q < n; ++q) used[q] += Align128(std::max<int64_t>(0, std::min(len, it.cnt[q] - w0)) * esz);
      w0 += len;
    }
  }
  flush();
  return Status::OK();
}

// A fused allgather response is ONE exchange launch while the blocks fit: every rank packs its blocks of all tensors back
// to back into its symmetric buffer and pulls every peer's blocks straight into the output tensors.  A tensor with a block
// larger than the buffer runs alone, in windows of the buffer's size.
Status PlanAllgather(int me, int n, const std::vector<PlanTensor>& ts, int64_t esz, int64_t cap, int comm_ctas, Plan* plan) {
  cap = cap / 16 * 16;
  if (cap <= 0) return Status::InvalidArgument("allgather: a symmetric buffer of " + Str(cap) + " bytes cannot hold 16 bytes");
  struct Item { const PlanTensor* t; std::vector<int64_t> bytes, displ; };
  std::vector<Item> items(ts.size());
  for (size_t ti = 0; ti < ts.size(); ++ti) {
    Item& it = items[ti];
    it.t = &ts[ti]; it.bytes.assign(n, 0); it.displ.assign(n + 1, 0);
    for (int p = 0; p < n; ++p) {
      it.bytes[p] = ts[ti].dims[p] * ts[ti].row * esz;
      it.displ[p + 1] = it.displ[p] + it.bytes[p];
    }
  }
  // segment = tensors whose blocks fit together in every rank's symmetric buffer
  std::vector<kern::CopyDesc> sends, recvs;
  std::vector<int64_t> used(n, 0);
  auto flush = [&]() {
    if (!sends.empty() || !recvs.empty()) AddExchange(plan, sends, recvs, comm_ctas, *std::max_element(used.begin(), used.end()));
    sends.clear(); recvs.clear(); used.assign(n, 0);
  };
  for (auto& it : items) {
    const int64_t maxb = *std::max_element(it.bytes.begin(), it.bytes.end());
    if (maxb > cap) {
      // one tensor larger than the buffer: windows of `cap` bytes, each its own launch
      flush();
      for (int64_t w0 = 0; w0 < maxb; w0 += cap) {
        int64_t mine = std::max<int64_t>(0, std::min(cap, it.bytes[me] - w0));
        if (mine) sends.push_back({(const char*)it.t->in + w0, nullptr, 0, mine, me, 0});
        for (int k = 0; k < n; ++k) {
          int p = (me + k) % n;
          int64_t b = std::max<int64_t>(0, std::min(cap, it.bytes[p] - w0));
          if (b) recvs.push_back({nullptr, (char*)it.t->out + it.displ[p] + w0, 0, b, p, 0});
          used[p] = b;
        }
        flush();
      }
      continue;
    }
    bool fits = true;
    for (int p = 0; p < n; ++p) if (used[p] + Align16(it.bytes[p]) > cap) fits = false;
    if (!fits) flush();
    if (it.bytes[me]) sends.push_back({it.t->in, nullptr, used[me], it.bytes[me], me, 0});
    for (int k = 0; k < n; ++k) {
      int p = (me + k) % n;  // start at my own block and rotate: at any instant the N ranks pull from N different peers
      if (it.bytes[p]) recvs.push_back({nullptr, (char*)it.t->out + it.displ[p], used[p], it.bytes[p], p, 0});
    }
    for (int p = 0; p < n; ++p) used[p] += Align16(it.bytes[p]);
  }
  flush();
  return Status::OK();
}

// Broadcast responses of one root are fused by the controller; a fused response is ONE launch while it fits.  With
// multicast the root stores through the multicast mapping (multimem.st: one source read, one egress stream, the switch
// replicates) and every rank copies out of its OWN buffer; without it the peers pull from the root's buffer.
Status PlanBroadcast(int me, int n, int root, const std::vector<PlanTensor>& ts, bool multicast, int64_t cap, int comm_ctas,
                     Plan* plan) {
  (void)n;
  cap = cap / 16 * 16;
  if (cap <= 0) return Status::InvalidArgument("broadcast: a symmetric buffer of " + Str(cap) + " bytes cannot hold 16 bytes");
  std::vector<kern::CopyDesc> sends, recvs;
  int64_t used = 0;
  auto flush = [&]() {
    if (used == 0) return;
    AddExchange(plan, sends, recvs, comm_ctas, used);
    sends.clear(); recvs.clear(); used = 0;
  };
  auto add = [&](const char* in, char* out, int64_t b) {
    if (me == root) sends.push_back({in, nullptr, used, b, me, multicast ? kern::kSendMulticast : 0});
    if (me != root || (out && out != in)) recvs.push_back({nullptr, out, used, b, multicast ? me : root, 0});
    used += Align16(b);
  };
  for (auto& t : ts) {
    const int64_t bytes = t.dims[0];
    if (bytes == 0) continue;
    for (int64_t w0 = 0; w0 < bytes; ) {
      if (cap - used < 16) flush();
      const int64_t b = std::min(cap - used, bytes - w0);
      add((const char*)t.in + w0, t.out ? (char*)t.out + w0 : nullptr, b);
      w0 += b;
    }
  }
  flush();
  return Status::OK();
}

// Window scheme, one tensor at a time: destination q's block occupies [q*win, (q+1)*win) of the sender's buffer; blocks
// larger than `win` take several launches.
Status PlanAlltoall(int me, int n, const std::vector<PlanTensor>& ts, int64_t esz, int64_t cap, int comm_ctas, Plan* plan) {
  for (auto& t : ts) {
    std::vector<int64_t> sbytes(n), rbytes(n), sdisp(n + 1, 0), rdisp(n + 1, 0);
    int64_t maxblock = 0;
    for (int p = 0; p < n; ++p) {
      sbytes[p] = t.dims[(size_t)me * n + p] * t.row * esz;
      rbytes[p] = t.dims[(size_t)p * n + me] * t.row * esz;
      sdisp[p + 1] = sdisp[p] + sbytes[p];
      rdisp[p + 1] = rdisp[p] + rbytes[p];
    }
    for (size_t i = 0; i < (size_t)n * n; ++i) maxblock = std::max(maxblock, t.dims[i] * t.row * esz);
    if (maxblock == 0) continue;  // nothing moves on any rank
    const int64_t win = std::min<int64_t>((maxblock + 15) / 16 * 16, cap / n / 16 * 16);
    if (win <= 0)
      return Status::InvalidArgument("alltoall: a symmetric buffer of " + Str(cap) + " bytes has no 16-byte window for each of " +
                                     Str(n) + " ranks");
    for (int64_t w0 = 0; w0 < maxblock; w0 += win) {
      std::vector<kern::CopyDesc> sends, recvs;
      for (int q = 0; q < n; ++q) {
        int64_t b = std::max<int64_t>(0, std::min(win, sbytes[q] - w0));
        if (b) sends.push_back({(const char*)t.in + sdisp[q] + w0, nullptr, q * win, b, me, 0});
      }
      for (int k = 0; k < n; ++k) {
        int p = (me + k) % n;
        int64_t b = std::max<int64_t>(0, std::min(win, rbytes[p] - w0));
        if (b) recvs.push_back({nullptr, (char*)t.out + rdisp[p] + w0, me * win, b, p, 0});
      }
      AddExchange(plan, sends, recvs, comm_ctas, std::min<int64_t>(maxblock - w0, win) * n);
    }
  }
  return Status::OK();
}

// ---------------------------------------------------------------------------

namespace {
Status Bad(size_t k, int r, const std::string& what) {
  return Status::InvalidArgument("launch " + Str((int64_t)k) + " rank " + Str(r) + ": " + what);
}
uintptr_t U(const void* p) { return (uintptr_t)p; }

Status CheckReduce(const std::vector<Plan>& plans, size_t k, int64_t cap) {
  const int n = (int)plans.size();
  const kern::AllreduceArgs& a0 = plans[0][k].args;
  const int64_t wsz = (int64_t)DataTypeSize((DataType)a0.wire_dtype);
  const int64_t T = a0.total_bytes;
  if (T <= 0 || T > cap || T % n) return Bad(k, 0, "total_bytes " + Str(T) + " is not n regions inside the buffer of " + Str(cap));
  const int64_t W = T / n;
  if (W % 128) return Bad(k, 0, "region width " + Str(W) + " is not a multiple of 128");
  if (a0.ndesc % n) return Bad(k, 0, "in-descriptors are not n regions");
  const int per = a0.ndesc / n;
  for (int r = 0; r < n; ++r) {
    const PlanLaunch& l = plans[r][k];
    const kern::AllreduceArgs& a = l.args;
    if (a.ndesc != a0.ndesc || a.nout != a0.nout || a.total_bytes != a0.total_bytes || a.op != a0.op || a.dtype != a0.dtype ||
        a.wire_dtype != a0.wire_dtype || a.variant != a0.variant || a.prescale != a0.prescale || a.postscale != a0.postscale ||
        a.oneshot_nvls != a0.oneshot_nvls)
      return Bad(k, r, "reduce arguments differ from rank 0's");
    if (a.variant != kern::kOneShot) return Bad(k, r, "not a one-shot reduce");
    if (a.nout != per) return Bad(k, r, "nout " + Str(a.nout) + " != descriptors per region " + Str(per));
    if ((int64_t)l.table.size() != (int64_t)a.ndesc + a.nout) return Bad(k, r, "table size");
    for (int i = 0; i < a.ndesc; ++i) {
      const kern::TensorDesc& d = l.table[i];
      const kern::TensorDesc& d0 = plans[0][k].table[i];
      if (d.offset != d0.offset || d.count != d0.count) return Bad(k, r, "packed layout differs from rank 0's at in-desc " + Str(i));
      const int q = i / per;
      const int64_t next = (i + 1 < a.ndesc) ? l.table[i + 1].offset : T;
      if (d.count < 0 || d.offset % 128 || d.offset < (int64_t)q * W || d.offset + d.count * wsz > (int64_t)(q + 1) * W ||
          d.offset + d.count * wsz > next || next < d.offset)
        return Bad(k, r, "in-desc " + Str(i) + " [" + Str(d.offset) + ", +" + Str(d.count * wsz) + ") is not in order inside region " +
                         Str(q));
    }
    if (a.reduce_lo != (int64_t)r * W || a.reduce_hi < a.reduce_lo || a.reduce_hi > (int64_t)(r + 1) * W)
      return Bad(k, r, "[reduce_lo, reduce_hi) = [" + Str(a.reduce_lo) + ", " + Str(a.reduce_hi) + ") is not inside region " + Str(r));
    for (int j = 0; j < a.nout; ++j) {
      const kern::TensorDesc& o = l.table[a.ndesc + j];
      const kern::TensorDesc& in = l.table[r * per + j];
      if (o.offset != in.offset || o.count != in.count)
        return Bad(k, r, "out-desc " + Str(j) + " does not sit on region " + Str(r) + "'s in-desc");
      if (o.offset + o.count * wsz > a.reduce_hi) return Bad(k, r, "out-desc " + Str(j) + " ends past reduce_hi");
    }
  }
  return Status::OK();
}

Status CheckExchange(const std::vector<Plan>& plans, size_t k, int64_t cap, int root) {
  const int n = (int)plans.size();
  // every rank's sends, sorted by offset; multicast sends land in every rank's buffer
  std::vector<std::vector<kern::CopyDesc>> sends(n);
  std::vector<kern::CopyDesc> mc;
  for (int r = 0; r < n; ++r) {
    for (const kern::CopyDesc& s : plans[r][k].sends) {
      if (s.bytes <= 0 || s.offset < 0 || s.offset % 16 || s.offset + s.bytes > cap)
        return Bad(k, r, "send [" + Str(s.offset) + ", +" + Str(s.bytes) + ") is not a 16 B aligned range inside [0, " + Str(cap) + ")");
      (s.pad == kern::kSendMulticast ? mc : sends[r]).push_back(s);
    }
    auto by_off = [](const kern::CopyDesc& x, const kern::CopyDesc& y) { return x.offset < y.offset; };
    std::sort(sends[r].begin(), sends[r].end(), by_off);
    for (size_t i = 1; i < sends[r].size(); ++i)
      if (sends[r][i - 1].offset + sends[r][i - 1].bytes > sends[r][i].offset) return Bad(k, r, "two sends overlap in the buffer");
  }
  for (int r = 0; r < n; ++r) {
    for (const kern::CopyDesc& d : plans[r][k].recvs) {
      if (d.bytes <= 0 || d.offset < 0 || d.offset % 16 || d.offset + d.bytes > cap || d.peer < 0 || d.peer >= n)
        return Bad(k, r, "recv [" + Str(d.offset) + ", +" + Str(d.bytes) + ") from peer " + Str(d.peer) + " is out of range");
      bool found = false;
      for (const kern::CopyDesc& s : mc) found = found || (s.offset <= d.offset && d.offset + d.bytes <= s.offset + s.bytes);
      if (!found) {
        if (root >= 0 && d.peer != root) return Bad(k, r, "broadcast recv from " + Str(d.peer) + ", not from the root");
        const auto& ss = sends[d.peer];
        auto it = std::upper_bound(ss.begin(), ss.end(), d.offset, [](int64_t o, const kern::CopyDesc& s) { return o < s.offset; });
        found = it != ss.begin() && std::prev(it)->offset + std::prev(it)->bytes >= d.offset + d.bytes;
      }
      if (!found) return Bad(k, r, "recv [" + Str(d.offset) + ", +" + Str(d.bytes) + ") from peer " + Str(d.peer) + " matches no send");
    }
  }
  return Status::OK();
}
}  // namespace

Status CheckPlans(const std::vector<Plan>& plans, const std::vector<std::vector<OutSpan>>& outputs, int64_t cap, int root) {
  const int n = (int)plans.size();
  if (n < 1 || (int)outputs.size() != n) return Status::InvalidArgument("CheckPlans: one plan and one output list per rank");
  for (int r = 1; r < n; ++r)
    if (plans[r].size() != plans[0].size())
      return Status::InvalidArgument("rank " + Str(r) + " plans " + Str((int64_t)plans[r].size()) + " launches, rank 0 " +
                                     Str((int64_t)plans[0].size()));
  for (size_t k = 0; k < plans[0].size(); ++k) {
    for (int r = 0; r < n; ++r) {
      const PlanLaunch& l = plans[r][k];
      if (l.reduce != plans[0][k].reduce || l.ctas != plans[0][k].ctas) return Bad(k, r, "kind or ctas differ from rank 0's");
      if (l.ctas < 1 || l.ctas > kern::kMaxCtas) return Bad(k, r, "ctas " + Str(l.ctas) + " out of range");
    }
    Status st = plans[0][k].reduce ? CheckReduce(plans, k, cap) : CheckExchange(plans, k, cap, root);
    if (!st.ok()) return st;
  }
  // coverage: the written byte ranges of each rank tile its outputs exactly
  for (int r = 0; r < n; ++r) {
    std::vector<std::pair<uintptr_t, uintptr_t>> w, want;
    for (const PlanLaunch& l : plans[r]) {
      if (l.reduce) {
        const int64_t tsz = (int64_t)DataTypeSize((DataType)l.args.dtype);
        for (int j = 0; j < l.args.nout; ++j) {
          const kern::TensorDesc& o = l.table[l.args.ndesc + j];
          if (o.count > 0) w.push_back({U(o.out), U(o.out) + (uintptr_t)(o.count * tsz)});
        }
      } else {
        for (const kern::CopyDesc& d : l.recvs) w.push_back({U(d.dst), U(d.dst) + (uintptr_t)d.bytes});
      }
    }
    for (const OutSpan& s : outputs[r]) if (s.bytes > 0) want.push_back({U(s.p), U(s.p) + (uintptr_t)s.bytes});
    std::sort(w.begin(), w.end());
    std::sort(want.begin(), want.end());
    auto merge = [](std::vector<std::pair<uintptr_t, uintptr_t>>& v, bool strict) -> bool {
      std::vector<std::pair<uintptr_t, uintptr_t>> m;
      for (auto& x : v) {
        if (!m.empty() && x.first < m.back().second) { if (strict) return false; m.back().second = std::max(m.back().second, x.second); }
        else if (!m.empty() && x.first == m.back().second) m.back().second = x.second;
        else m.push_back(x);
      }
      v.swap(m);
      return true;
    };
    if (!merge(w, true)) return Status::InvalidArgument("rank " + Str(r) + ": an output byte is written twice");
    merge(want, false);
    if (w != want) return Status::InvalidArgument("rank " + Str(r) + ": the written ranges do not cover the outputs exactly");
  }
  return Status::OK();
}

}  // namespace hvd
