// In-process unit tests of the native runtime, callable through ctypes
// (tests/test_native_unit.py).  Several Engine instances run in ONE process on
// the loopback transport, so negotiation, caching, fusion, join and the CPU
// collectives are exercised without any launcher — the reference has no
// equivalent (all its multi-rank tests need real MPI/Gloo processes).
#include <atomic>
#include <chrono>
#include <condition_variable>
#include <mutex>
#include <map>
#include <cmath>
#include <cstdio>
#include <future>
#include <sstream>
#include <thread>
#include <cstdlib>
#include <unistd.h>
#include "../ops/cpu_ops.h"
#include "../transport/transport.h"
#include "controller.h"
#include "engine.h"
#include "half.h"
#include "message.h"
#include "optim/bayesian_optimization.h"
#include "parameter_manager.h"
#include "response_cache.h"

using namespace hvd;

namespace {
int g_failures = 0;
std::ostringstream g_log;
#define CHECK_T(cond)                                                                     \
  do {                                                                                    \
    if (!(cond)) { ++g_failures; g_log << __FILE__ << ":" << __LINE__ << " CHECK failed: " #cond "\n"; } \
  } while (0)

Response MkResp(const std::string& name, int64_t n, DataType dt = DataType::FLOAT32, int32_t group = -1) {
  Response r;
  r.type = ResponseType::ALLREDUCE; r.tensor_names = {name}; r.tensor_sizes = {n}; r.dtype = dt; r.devices = {-1, -1};
  r.group_id = group;
  return r;
}

void TestWire() {
  RequestList rl;
  Request q; q.request_rank = 3; q.type = RequestType::ALLGATHER; q.dtype = DataType::BFLOAT16; q.name = "x.y"; q.root_rank = 2;
  q.device = 5; q.shape = {7, 8, 9}; q.prescale = 0.5; q.postscale = 2.0; q.reduce_op = ReduceOp::MAX; q.group_id = 4; q.group_size = 6;
  rl.requests.push_back(q); rl.shutdown = true;
  auto bytes = rl.Serialize();
  RequestList back = RequestList::Parse(bytes.data(), bytes.size());
  CHECK_T(back.shutdown && back.requests.size() == 1);
  const Request& b = back.requests[0];
  CHECK_T(b.request_rank == 3 && b.type == RequestType::ALLGATHER && b.dtype == DataType::BFLOAT16 && b.name == "x.y");
  CHECK_T(b.shape == q.shape && b.prescale == 0.5 && b.postscale == 2.0 && b.reduce_op == ReduceOp::MAX && b.group_size == 6);
  ResponseList sl;
  Response r = MkResp("t", 10); r.error_message = "boom"; r.last_joined_rank = 1;
  sl.responses.push_back(r);
  auto sb = sl.Serialize();
  ResponseList sback = ResponseList::Parse(sb.data(), sb.size());
  CHECK_T(sback.responses.size() == 1 && sback.responses[0].error_message == "boom" && sback.responses[0].tensor_sizes[0] == 10);
  bool threw = false;
  try { RequestList::Parse(bytes.data(), bytes.size() / 2); } catch (const std::exception&) { threw = true; }
  CHECK_T(threw);
}

void TestHalf() {
  for (float v : {0.0f, 1.0f, -2.5f, 65504.0f, 1e-5f, 3.14159f, -1e-8f}) {
    float h = HalfBitsToFloat(FloatToHalfBits(v));
    CHECK_T(std::fabs(h - v) <= std::fabs(v) * 1e-3f + 1e-7f);
    float b = BF16BitsToFloat(FloatToBF16Bits(v));
    CHECK_T(std::fabs(b - v) <= std::fabs(v) * 8e-3f + 1e-30f);
  }
  CHECK_T(std::isinf(HalfBitsToFloat(FloatToHalfBits(1e6f))));
}

void TestFusion() {
  std::deque<Response> in;
  for (int i = 0; i < 6; ++i) in.push_back(MkResp("f" + std::to_string(i), 1000));
  auto out = Controller::FuseResponses(in, 1 << 20, false);
  CHECK_T(out.size() == 1 && out[0].tensor_names.size() == 6);
  // threshold: 1000 floats = 4000 B -> padded 4096; threshold 9000 fits two
  out = Controller::FuseResponses(in, 9000, false);
  CHECK_T(out.size() == 3 && out[0].tensor_names.size() == 2);
  // threshold 0 disables fusion
  out = Controller::FuseResponses(in, 0, false);
  CHECK_T(out.size() == 6);
  // look-ahead across a dtype change keeps order within each dtype
  std::deque<Response> mixed;
  mixed.push_back(MkResp("a0", 10));
  mixed.push_back(MkResp("h0", 10, DataType::FLOAT16));
  mixed.push_back(MkResp("a1", 10));
  mixed.push_back(MkResp("h1", 10, DataType::FLOAT16));
  out = Controller::FuseResponses(mixed, 1 << 20, false);
  CHECK_T(out.size() == 2);
  CHECK_T(out[0].tensor_names == std::vector<std::string>({"a0", "a1"}));
  CHECK_T(out[1].tensor_names == std::vector<std::string>({"h0", "h1"}));
  // group fusion disabled: groups do not merge with others
  std::deque<Response> grouped;
  grouped.push_back(MkResp("g0", 10, DataType::FLOAT32, 1));
  grouped.push_back(MkResp("g1", 10, DataType::FLOAT32, 1));
  grouped.push_back(MkResp("u0", 10, DataType::FLOAT32, -1));
  out = Controller::FuseResponses(grouped, 1 << 20, true);
  CHECK_T(out.size() == 2 && out[0].tensor_names.size() == 2);
  out = Controller::FuseResponses(grouped, 1 << 20, false);
  CHECK_T(out.size() == 1);
  // allgather fuses (per-rank first dims are concatenated tensor by tensor) up to the threshold on its output bytes
  std::deque<Response> ag;
  Response g = MkResp("ag0", 4); g.type = ResponseType::ALLGATHER; g.tensor_sizes = {2, 5}; g.payload_bytes = 256; ag.push_back(g);
  g.tensor_names = {"ag1"}; g.tensor_sizes = {3, 1}; ag.push_back(g);
  out = Controller::FuseResponses(ag, 1 << 20, false);
  CHECK_T(out.size() == 1 && out[0].tensor_sizes == std::vector<int64_t>({2, 5, 3, 1}) && out[0].payload_bytes == 512);
  CHECK_T(Controller::FuseResponses(ag, 300, false).size() == 2);
  // reducescatter fuses with the allreduce rule; broadcasts fuse only when they share the root
  std::deque<Response> rs;
  Response q = MkResp("rs0", 100); q.type = ResponseType::REDUCESCATTER; rs.push_back(q);
  q.tensor_names = {"rs1"}; rs.push_back(q);
  CHECK_T(Controller::FuseResponses(rs, 1 << 20, false).size() == 1);
  std::deque<Response> bc;
  Response b0 = MkResp("b0", 100); b0.type = ResponseType::BROADCAST; b0.root_rank = 0; bc.push_back(b0);
  Response b1 = MkResp("b1", 100); b1.type = ResponseType::BROADCAST; b1.root_rank = 1; bc.push_back(b1);
  Response b2 = MkResp("b2", 100); b2.type = ResponseType::BROADCAST; b2.root_rank = 0; bc.push_back(b2);
  out = Controller::FuseResponses(bc, 1 << 20, false);
  CHECK_T(out.size() == 2 && out[0].tensor_names == std::vector<std::string>({"b0", "b2"}));
}

void TestValidation() {
  auto mk = [](int rank, std::vector<int64_t> shape, DataType dt = DataType::FLOAT32, RequestType t = RequestType::ALLREDUCE) {
    Request q; q.request_rank = rank; q.type = t; q.dtype = dt; q.name = "v"; q.shape = std::move(shape); q.device = -1; return q;
  };
  Response r = Controller::ConstructResponse("v", {mk(0, {4}), mk(1, {4})}, 2, {});
  CHECK_T(r.type == ResponseType::ALLREDUCE && r.tensor_sizes[0] == 4);
  r = Controller::ConstructResponse("v", {mk(0, {4}), mk(1, {5})}, 2, {});
  CHECK_T(r.type == ResponseType::ERROR && r.error_message.find("shape") != std::string::npos);
  r = Controller::ConstructResponse("v", {mk(0, {4}), mk(1, {4}, DataType::FLOAT64)}, 2, {});
  CHECK_T(r.type == ResponseType::ERROR && r.error_message.find("data types") != std::string::npos);
  Request a = mk(0, {4}), b = mk(1, {4}); b.prescale = 2.0;
  CHECK_T(Controller::ConstructResponse("v", {a, b}, 2, {}).type == ResponseType::ERROR);
  b = mk(1, {4}); b.device = 0;
  CHECK_T(Controller::ConstructResponse("v", {a, b}, 2, {}).error_message.find("CPU/GPU") != std::string::npos);
  // allgather: first dim may differ, others not
  r = Controller::ConstructResponse("v", {mk(0, {2, 3}, DataType::FLOAT32, RequestType::ALLGATHER), mk(1, {5, 3}, DataType::FLOAT32, RequestType::ALLGATHER)}, 2, {});
  CHECK_T(r.type == ResponseType::ALLGATHER && r.tensor_sizes == std::vector<int64_t>({2, 5}));
  r = Controller::ConstructResponse("v", {mk(0, {2, 3}, DataType::FLOAT32, RequestType::ALLGATHER), mk(1, {2, 4}, DataType::FLOAT32, RequestType::ALLGATHER)}, 2, {});
  CHECK_T(r.type == ResponseType::ERROR);
  // join is incompatible with allgather
  r = Controller::ConstructResponse("v", {mk(0, {2, 3}, DataType::FLOAT32, RequestType::ALLGATHER)}, 2, {1});
  CHECK_T(r.type == ResponseType::ERROR && r.error_message.find("Join") != std::string::npos);
  // broadcast root mismatch
  Request b0 = mk(0, {4}, DataType::FLOAT32, RequestType::BROADCAST), b1 = mk(1, {4}, DataType::FLOAT32, RequestType::BROADCAST);
  b1.root_rank = 1;
  CHECK_T(Controller::ConstructResponse("v", {b0, b1}, 2, {}).error_message.find("root") != std::string::npos);
  // zero-copy keys: registered region only if identical everywhere; IPC (-2) only if EVERY rank offers a plain-allocation key
  Request z0 = mk(0, {1024}), z1 = mk(1, {1024});
  z0.device = z1.device = 0;
  z0.symm_key = z1.symm_key = (3ll << 44) | 4096;
  CHECK_T(Controller::ConstructResponse("v", {z0, z1}, 2, {}).symm_key == ((3ll << 44) | 4096));
  z1.symm_key = (3ll << 44) | 8192;
  CHECK_T(Controller::ConstructResponse("v", {z0, z1}, 2, {}).symm_key == -1);
  z0.symm_key = -12345; z1.symm_key = -99;   // per-rank IPC keys differ by construction
  CHECK_T(Controller::ConstructResponse("v", {z0, z1}, 2, {}).symm_key == -2);
  z1.symm_key = -1;                          // one rank cannot export its tensor
  CHECK_T(Controller::ConstructResponse("v", {z0, z1}, 2, {}).symm_key == -1);
  z1.symm_key = -99;
  CHECK_T(Controller::ConstructResponse("v", {z0}, 2, {1}).symm_key == -1);  // a joined rank has no tensor to register
  // a response that carries a zero-copy key is never fused with its neighbours
  {
    std::deque<Response> zs;
    Response a = MkResp("za", 1 << 20), b = MkResp("zb", 1 << 20), c = MkResp("zc", 1 << 20);
    b.symm_key = -2;
    zs.push_back(a); zs.push_back(b); zs.push_back(c);
    auto fused = Controller::FuseResponses(zs, 1ll << 30, false);
    CHECK_T(fused.size() == 2 && fused[0].tensor_names == std::vector<std::string>({"za", "zc"}) && fused[1].symm_key == -2);
  }
  // alltoall without explicit splits: "uniform" only when NO rank gave splits and every rank sends the same number of rows
  Request a0 = mk(0, {8, 2}, DataType::FLOAT32, RequestType::ALLTOALL), a1 = mk(1, {8, 2}, DataType::FLOAT32, RequestType::ALLTOALL);
  a0.root_rank = a1.root_rank = kUniformSplits;
  CHECK_T(Controller::ConstructResponse("v", {a0, a1}, 2, {}).root_rank == kUniformSplits);
  a1.root_rank = 0;  // explicit splits on one rank
  CHECK_T(Controller::ConstructResponse("v", {a0, a1}, 2, {}).root_rank == 0);
  a1.root_rank = kUniformSplits; a1.shape = {12, 2};  // different dim 0
  CHECK_T(Controller::ConstructResponse("v", {a0, a1}, 2, {}).root_rank == 0);
}

void TestCache() {
  ResponseCache c;
  c.set_capacity(3);
  auto req = [](const std::string& n, int64_t len) { Request q; q.name = n; q.shape = {len}; q.dtype = DataType::FLOAT32; q.device = -1; return q; };
  for (int i = 0; i < 3; ++i) { Request q = req("t" + std::to_string(i), 8); CHECK_T(c.Put(MkResp(q.name, 8), &q) == UINT32_MAX); }
  CHECK_T(c.Cached(req("t0", 8)) == ResponseCache::State::HIT);
  CHECK_T(c.Cached(req("t0", 9)) == ResponseCache::State::INVALID);
  CHECK_T(c.Cached(req("zz", 8)) == ResponseCache::State::MISS);
  c.GetResponse(c.PeekBit("t0"));  // t0 becomes most recently used -> t1 is the LRU victim
  Request q3 = req("t3", 8);
  uint32_t ev = c.Put(MkResp("t3", 8), &q3);
  CHECK_T(ev != UINT32_MAX);
  CHECK_T(c.Cached(req("t1", 8)) == ResponseCache::State::MISS);
  CHECK_T(c.Cached(req("t0", 8)) == ResponseCache::State::HIT);
  CHECK_T(c.PeekBit("t3") == ev);  // slot reuse keeps bit numbering dense
  // a slot stored without local parameters (joined rank) never hits
  c.Put(MkResp("j", 8), nullptr);
  CHECK_T(c.Cached(req("j", 8)) == ResponseCache::State::INVALID);
}

void TestCpuOps(int n) {
  auto hub = CreateLoopbackHub(n);
  std::vector<std::thread> th;
  std::atomic<int> bad{0};
  for (int r = 0; r < n; ++r) {
    th.emplace_back([&, r] {
      auto t = LoopbackEndpoint(hub, r);
      // ring allreduce (large) and star allreduce (small)
      for (int64_t cnt : {5, 100003}) {
        std::vector<float> v(cnt);
        for (int64_t i = 0; i < cnt; ++i) v[i] = (float)(r + 1) * (float)(i % 7);
        cpu::Allreduce(t.get(), v.data(), cnt, DataType::FLOAT32, ReduceOp::SUM);
        float tot = (float)n * (n + 1) / 2;
        for (int64_t i = 0; i < cnt; ++i) if (std::fabs(v[i] - tot * (float)(i % 7)) > 1e-3f) { bad++; break; }
      }
      // allgatherv
      std::vector<int64_t> bytes(n);
      int64_t total = 0;
      for (int p = 0; p < n; ++p) { bytes[p] = (p + 1) * 3; total += bytes[p]; }
      std::vector<char> mine(bytes[r], (char)('a' + r)), all(total);
      cpu::Allgatherv(t.get(), mine.data(), all.data(), bytes);
      int64_t off = 0;
      for (int p = 0; p < n; ++p) { for (int64_t i = 0; i < bytes[p]; ++i) if (all[off + i] != (char)('a' + p)) bad++; off += bytes[p]; }
      // broadcast from every root
      for (int root = 0; root < n; ++root) { int64_t x = r == root ? 4242 + root : -1; cpu::Broadcast(t.get(), &x, 8, root); if (x != 4242 + root) bad++; }
      // alltoallv: rank r sends (d+1) ints with value r*100+d to d
      std::vector<int64_t> sb(n), rb(n);
      std::vector<int32_t> send, recv((size_t)n * (r + 1));
      for (int d = 0; d < n; ++d) { sb[d] = (d + 1) * 4; rb[d] = (r + 1) * 4; for (int k = 0; k <= d; ++k) send.push_back(r * 100 + d); }
      cpu::Alltoallv(t.get(), send.data(), sb, recv.data(), rb);
      for (int p = 0; p < n; ++p) for (int k = 0; k <= r; ++k) if (recv[(size_t)p * (r + 1) + k] != p * 100 + r) bad++;
      // reducescatter with uneven counts
      std::vector<int64_t> counts(n);
      int64_t tc = 0;
      for (int p = 0; p < n; ++p) { counts[p] = 2 + (p == 0 ? 1 : 0); tc += counts[p]; }
      std::vector<double> buf(tc), out(counts[r]);
      for (int64_t i = 0; i < tc; ++i) buf[i] = (double)(r + 1) + i;
      cpu::Reducescatter(t.get(), buf.data(), counts, out.data(), DataType::FLOAT64, ReduceOp::SUM);
      int64_t o = 0;
      for (int p = 0; p < r; ++p) o += counts[p];
      for (int64_t i = 0; i < counts[r]; ++i) if (std::fabs(out[i] - ((double)n * (n + 1) / 2 + (double)n * (o + i))) > 1e-9) bad++;
    });
  }
  for (auto& t : th) t.join();
  CHECK_T(bad.load() == 0);
}

// AND / OR reduction of bit vectors among a subset of ranks: star for small groups, recursive doubling (with the fold-in of the
// members beyond the largest power of two) otherwise.  HVD_BITS_TREE_MIN_RANKS is read once per process, so the selftest driver
// (tests/test_native_unit.py) runs this binary a second time with the knob at 2.
void TestBitsAmong(int n) {
  auto hub = CreateLoopbackHub(n);
  std::vector<std::thread> th;
  std::atomic<int> bad{0};
  for (int r = 0; r < n; ++r) {
    th.emplace_back([&, r] {
      auto t = LoopbackEndpoint(hub, r);
      // all ranks
      uint64_t a[2] = {~0ull & ~(1ull << r), 0xF0F0ull}, o[1] = {1ull << (r + 8)};
      t->AllreduceBits(a, 2, o, 1);
      uint64_t want_a = ~0ull, want_o = 0;
      for (int p = 0; p < n; ++p) { want_a &= ~(1ull << p); want_o |= 1ull << (p + 8); }
      if (a[0] != want_a || a[1] != 0xF0F0ull || o[0] != want_o) bad++;
      // the odd ranks only, listed in reverse order (positions, not ranks, drive the exchange pattern)
      std::vector<int> odd;
      for (int p = n - 1; p >= 0; --p) if (p & 1) odd.push_back(p);
      if ((r & 1) && odd.size() > 1) {
        int me = 0;
        while (odd[me] != r) ++me;
        uint64_t w[2] = {~(1ull << r), (uint64_t)r};
        t->AllreduceBitsAmong(odd, me, w, 1, 2);
        uint64_t wa = ~0ull, wo = 0;
        for (int p : odd) { wa &= ~(1ull << p); wo |= (uint64_t)p; }
        if (w[0] != wa || w[1] != wo) bad++;
      }
      t->Barrier();
    });
  }
  for (auto& t : th) t.join();
  CHECK_T(bad.load() == 0);
}

// The shared-memory control + data plane with the "ranks" being threads of this process (each maps the segments itself, like a
// process would): multi-piece allreduce, destination-major reducescatter, both regimes of the slot alltoall (everything in one
// slot / rotation rounds with ragged blocks), allgatherv and broadcast through slots of 8 KiB.  This is what puts
// shm_transport.cc and the Shm* collectives of cpu_ops.cc under the thread / address sanitizer builds.
void PlaneCollectives(Transport* tp, int n, int r, std::atomic<int>& bad) {
  Transport* t = tp;
  // bit vectors + barrier through the segment
  uint64_t a = ~(1ull << r), o = 1ull << r;
  t->AllreduceBits(&a, 1, &o, 1);
  uint64_t wa = ~0ull, wo = 0;
  for (int p = 0; p < n; ++p) { wa &= ~(1ull << p); wo |= 1ull << p; }
  if (a != wa || o != wo) bad++;
  // coordinator round: variable-length blobs to a root and one blob back; `big` makes one payload larger than an 8 KiB slot, which
  // sends every rank down the socket path together
  for (int big : {0, 1}) {
    for (int root : {0, n - 1}) {
      std::vector<uint8_t> mine((size_t)(10 + 37 * r + (big && r == n - 1 ? 20000 : 0)), (uint8_t)(r + 1));
      std::vector<std::vector<uint8_t>> all;
      t->GatherBytes(mine, &all, root);
      if (r == root) {
        if ((int)all.size() != n) bad++;
        else for (int p = 0; p < n; ++p) {
          const size_t want = (size_t)(10 + 37 * p + (big && p == n - 1 ? 20000 : 0));
          if (all[(size_t)p].size() != want || (want && (all[(size_t)p].front() != (uint8_t)(p + 1) || all[(size_t)p].back() != (uint8_t)(p + 1)))) bad++;
        }
      }
      std::vector<uint8_t> resp;
      if (r == root) resp.assign((size_t)(big ? 30000 : 123), (uint8_t)(200 + root % 50));
      t->BcastBytes(&resp, root);
      if (resp.size() != (size_t)(big ? 30000 : 123) || resp.front() != (uint8_t)(200 + root % 50) || resp.back() != (uint8_t)(200 + root % 50)) bad++;
    }
  }
  // integer tables (small: through the slots where there are some; larger than a slot's words: the star of the base transport)
  for (int per : {3, 700}) {
    std::vector<int64_t> mine_i((size_t)per), all_i((size_t)per * (size_t)n, -1);
    for (int i = 0; i < per; ++i) mine_i[(size_t)i] = (int64_t)r * 100000 + i;
    t->AllgatherInts(mine_i.data(), per, all_i.data());
    for (int p = 0; p < n; ++p) for (int i = 0; i < per; ++i) if (all_i[(size_t)p * (size_t)per + (size_t)i] != (int64_t)p * 100000 + i) { bad++; break; }
  }
  // allreduce over several pieces
  const int64_t cnt = 10007;
  std::vector<float> v(cnt);
  for (int64_t i = 0; i < cnt; ++i) v[i] = (float)(r + 1) * (float)(i % 5);
  cpu::Allreduce(t, v.data(), cnt, DataType::FLOAT32, ReduceOp::SUM);
  for (int64_t i = 0; i < cnt; ++i) if (std::fabs(v[i] - (float)(n * (n + 1) / 2) * (float)(i % 5)) > 1e-3f) { bad++; break; }
  // reducescatter, uneven segments, several steps
  std::vector<int64_t> counts(n);
  int64_t tc = 0;
  for (int p = 0; p < n; ++p) { counts[p] = 1500 + 700 * p; tc += counts[p]; }
  std::vector<double> buf(tc), out(counts[r]);
  for (int64_t i = 0; i < tc; ++i) buf[i] = (double)(r + 1) + (double)i;
  cpu::Reducescatter(t, buf.data(), counts, out.data(), DataType::FLOAT64, ReduceOp::SUM);
  int64_t off = 0;
  for (int p = 0; p < r; ++p) off += counts[p];
  for (int64_t i = 0; i < counts[r]; ++i) if (std::fabs(out[i] - ((double)n * (n + 1) / 2 + (double)n * (double)(off + i))) > 1e-6) { bad++; break; }
  // alltoall: k = 1 fits into one slot, k = 40 needs the rotation rounds; rank r sends (r + d) % 3 * k + (d ? 1 : 0) ints to d
  for (int k : {1, 40}) {
    std::vector<int64_t> sb(n), rb(n);
    std::vector<int32_t> send;
    for (int dst = 0; dst < n; ++dst) {
      const int64_t len = (int64_t)((r + dst) % 3) * 50 * k + (dst ? 1 : 0);
      sb[dst] = len * 4;
      for (int64_t i = 0; i < len; ++i) send.push_back(r * 1000 + dst * 10 + (int32_t)(i % 7));
    }
    int64_t rt = 0;
    for (int src = 0; src < n; ++src) { rb[src] = ((int64_t)((src + r) % 3) * 50 * k + (r ? 1 : 0)) * 4; rt += rb[src]; }
    std::vector<int32_t> recv((size_t)(rt / 4) + 1, -1);
    cpu::Alltoallv(t, send.data(), sb, recv.data(), rb);
    int64_t pos = 0;
    for (int src = 0; src < n; ++src)
      for (int64_t i = 0; i < rb[src] / 4; ++i, ++pos) if (recv[(size_t)pos] != src * 1000 + r * 10 + (int32_t)(i % 7)) { bad++; break; }
  }
  // allgatherv + broadcast from every root
  std::vector<int64_t> bytes(n);
  int64_t total = 0;
  for (int p = 0; p < n; ++p) { bytes[p] = 3000 * (p + 1) + 1; total += bytes[p]; }
  std::vector<char> mine(bytes[r], (char)('a' + r)), all(total);
  cpu::Allgatherv(t, mine.data(), all.data(), bytes);
  int64_t o2 = 0;
  for (int p = 0; p < n; ++p) { for (int64_t i = 0; i < bytes[p]; ++i) if (all[o2 + i] != (char)('a' + p)) { bad++; break; } o2 += bytes[p]; }
  for (int root = 0; root < n; ++root) {
    std::vector<int32_t> x(5000, r == root ? 77 + root : -1);
    cpu::Broadcast(t, x.data(), (int64_t)x.size() * 4, root);
    if (x.front() != 77 + root || x.back() != 77 + root) bad++;
  }
}

void TestShmPlane(int n) {
  if (n < 2) return;
  setenv("HVD_SHM_SLOT_BYTES", "8192", 1);
  static std::atomic<int> serial{0};
  const std::string seg = "hvd-selftest-" + std::to_string((long)getpid()) + "-" + std::to_string(serial.fetch_add(1));
  auto hub = CreateLoopbackHub(n);
  std::vector<std::thread> th;
  std::atomic<int> bad{0}, no_plane{0};
  for (int r = 0; r < n; ++r) {
    th.emplace_back([&, r] {
      std::shared_ptr<Transport> t = WrapWithShmControl(LoopbackEndpoint(hub, r), seg);
      ShmData d;
      if (!t->ShmDataPlane(&d)) { no_plane++; return; }               // no /dev/shm here: nothing to test
      PlaneCollectives(t.get(), n, r, bad);
      t->Barrier();
    });
  }
  for (auto& t : th) t.join();
  unsetenv("HVD_SHM_SLOT_BYTES");
  CHECK_T(bad.load() == 0);
  CHECK_T(no_plane.load() == 0 || no_plane.load() == n);
}

// A REAL socket mesh between the threads of this process (rendezvous through an in-memory KV store): the spinning receives, the
// all-peers-at-once alltoall, the chunk-pipelined ring with its reducer thread, the chunked chain broadcast and the log-depth
// bit reduction of tcp_transport.cc / transport.cc / cpu_ops.cc, so that they run under the sanitizer builds too.
class MemKVStore : public KVStore {
 public:
  void Set(const std::string& scope, const std::string& key, const std::string& value) override {
    std::lock_guard<std::mutex> l(m_);
    kv_[scope + "/" + key] = value;
    cv_.notify_all();
  }
  std::string Get(const std::string& scope, const std::string& key, double timeout_s) override {
    std::unique_lock<std::mutex> l(m_);
    const std::string k = scope + "/" + key;
    if (!cv_.wait_for(l, std::chrono::duration<double>(timeout_s), [&] { return kv_.count(k) > 0; }))
      throw TransportError("MemKVStore: timed out waiting for " + k);
    return kv_[k];
  }

 private:
  std::mutex m_;
  std::condition_variable cv_;
  std::map<std::string, std::string> kv_;
};

void TestTcpMesh(int n) {
  MemKVStore store;
  static std::atomic<int> serial{0};
  const std::string scope = "selftest.tcp." + std::to_string(serial.fetch_add(1));
  std::vector<std::thread> th;
  std::atomic<int> bad{0}, failed{0};
  for (int r = 0; r < n; ++r) {
    th.emplace_back([&, r] {
      std::shared_ptr<Transport> t;
      try {
        t = CreateTcpTransport(r, n, &store, scope, "127.0.0.1", 30.0);
      } catch (const std::exception& e) { failed++; return; }     // no loopback networking in this sandbox
      try {
        PlaneCollectives(t.get(), n, r, bad);
        // a long allreduce and a long broadcast: pipelined ring steps (when HVD_RING_CHUNK_BYTES is small) / chunked chain
        const int64_t cnt = 300007;
        std::vector<float> v(cnt);
        for (int64_t i = 0; i < cnt; ++i) v[i] = (float)(r + 1) * (float)(i % 3);
        cpu::Allreduce(t.get(), v.data(), cnt, DataType::FLOAT32, ReduceOp::SUM);
        for (int64_t i = 0; i < cnt; ++i) if (std::fabs(v[i] - (float)(n * (n + 1) / 2) * (float)(i % 3)) > 1e-3f) { bad++; break; }
        std::vector<int32_t> x(200003, r == n - 1 ? 4242 : -1);
        cpu::Broadcast(t.get(), x.data(), (int64_t)x.size() * 4, n - 1);
        if (x.front() != 4242 || x[100001] != 4242 || x.back() != 4242) bad++;
        t->Barrier();
      } catch (const std::exception& e) { bad++; }
    });
  }
  for (auto& t : th) t.join();
  CHECK_T(bad.load() == 0);
  CHECK_T(failed.load() == 0 || failed.load() == n);
}

// The two-level planes (shm inside a "host", loopback queues standing in for the sockets between hosts): hosts x per_host ranks.
void TestHierPlane(int hosts, int per_host) {
  const int n = hosts * per_host;
  setenv("HVD_SHM_SLOT_BYTES", "8192", 1);
  static std::atomic<int> serial{0};
  const std::string seg = "hvd-selftest-h-" + std::to_string((long)getpid()) + "-" + std::to_string(serial.fetch_add(1));
  std::vector<int> table((size_t)n);
  for (int r = 0; r < n; ++r) table[(size_t)r] = r / per_host;
  auto hub = CreateLoopbackHub(n);
  std::vector<std::thread> th;
  std::atomic<int> bad{0}, no_plane{0};
  for (int r = 0; r < n; ++r) {
    th.emplace_back([&, r] {
      std::shared_ptr<Transport> t = WrapWithHierarchicalControl(LoopbackEndpoint(hub, r, table), seg);
      HierData h;
      if (!t->HierDataPlane(&h)) { no_plane++; return; }
      if (h.local_size != per_host || (int)(*h.column)[0].size() != hosts) bad++;
      PlaneCollectives(t.get(), n, r, bad);
      t->Barrier();
    });
  }
  for (auto& t : th) t.join();
  unsetenv("HVD_SHM_SLOT_BYTES");
  CHECK_T(bad.load() == 0);
  CHECK_T(no_plane.load() == 0 || no_plane.load() == n);
}

void TestAdasum(int n) {
  if (n & (n - 1)) return;
  auto hub = CreateLoopbackHub(n);
  std::vector<std::thread> th;
  std::atomic<int> bad{0};
  for (int r = 0; r < n; ++r) {
    th.emplace_back([&, r] {
      auto t = LoopbackEndpoint(hub, r);
      // two fused tensors: #0 identical on all ranks (parallel -> stays the same), #1 orthogonal (-> sum)
      const int64_t c0 = 37, c1 = (int64_t)n * 5;
      std::vector<float> v(c0 + c1, 0.f);
      for (int64_t i = 0; i < c0; ++i) v[i] = (float)(i + 1);
      for (int64_t i = 0; i < 5; ++i) v[c0 + r * 5 + i] = (float)(r + 1);
      Status st = cpu::AdasumAllreduce(t.get(), v.data(), {c0, c1}, DataType::FLOAT32);
      if (!st.ok()) { bad++; return; }
      for (int64_t i = 0; i < c0; ++i) if (std::fabs(v[i] - (float)(i + 1)) > 1e-3f) { bad++; break; }
      for (int p = 0; p < n; ++p) for (int i = 0; i < 5; ++i) if (std::fabs(v[c0 + p * 5 + i] - (float)(p + 1)) > 1e-3f) { bad++; break; }
    });
  }
  for (auto& t : th) t.join();
  CHECK_T(bad.load() == 0);
}

// N engines on the loopback hub: negotiation, cache fast path, fusion, errors, join.
void TestEngines(int n, int planes = 0) {   // 0: loopback only, 1: one host's shm planes, 2: two-level planes (n / 2 "hosts" of 2 ranks)
  auto hub = CreateLoopbackHub(n);
  static std::atomic<int> serial{0};
  const std::string seg = "hvd-selftest-e-" + std::to_string((long)getpid()) + "-" + std::to_string(serial.fetch_add(1));
  std::vector<std::unique_ptr<Engine>> engines;
  for (int r = 0; r < n; ++r) engines.emplace_back(new Engine());
  std::vector<std::thread> th;
  std::atomic<int> bad{0};
  for (int r = 0; r < n; ++r) {
    th.emplace_back([&, r] {
      InitConfig cfg;
      cfg.rank = r; cfg.size = n; cfg.local_rank = r; cfg.local_size = n;
      // with shm_planes the engines negotiate and move host tensors the way the ranks of one host do (bit vectors, coordinator
      // round and data through the shared-memory segments)
      if (planes == 2) {
        std::vector<int> table((size_t)n);
        for (int q = 0; q < n; ++q) table[(size_t)q] = q / 2;
        cfg.transport = WrapWithHierarchicalControl(LoopbackEndpoint(hub, r, table), seg);
      } else {
        cfg.transport = planes == 1 ? WrapWithShmControl(LoopbackEndpoint(hub, r), seg) : LoopbackEndpoint(hub, r);
      }
      Engine& e = *engines[r];
      if (!e.Init(cfg).ok()) { bad++; return; }
      auto run_allreduce = [&](const std::string& name, std::vector<float>& v, ReduceOp op) -> Status {
        auto ent = std::make_shared<TensorTableEntry>();
        ent->name = name; ent->input = v.data(); ent->output = v.data(); ent->dtype = DataType::FLOAT32;
        ent->shape = TensorShape({(int64_t)v.size()}); ent->reduce_op = op;
        std::promise<Status> p;
        auto f = p.get_future();
        ent->callback = [&p](const Completion& c) { p.set_value(c.status); };
        std::vector<std::shared_ptr<TensorTableEntry>> es{ent};
        Status st = e.EnqueueAllreduces(es, 0);
        if (!st.ok()) return st;
        return f.get();
      };
      // repeated named allreduce: later rounds go through the response cache
      for (int step = 0; step < 5; ++step) {
        std::vector<float> v(64, (float)(r + 1));
        Status st = run_allreduce("cached", v, ReduceOp::AVERAGE);
        if (!st.ok() || std::fabs(v[0] - (float)(n + 1) / 2.f) > 1e-5f) bad++;
      }
      // many tensors at once -> fused
      {
        std::vector<std::vector<float>> bufs(20, std::vector<float>(100, (float)r));
        std::vector<std::promise<Status>> ps(20);
        for (int i = 0; i < 20; ++i) {
          auto ent = std::make_shared<TensorTableEntry>();
          ent->name = "many." + std::to_string(i); ent->input = bufs[i].data(); ent->output = bufs[i].data();
          ent->dtype = DataType::FLOAT32; ent->shape = TensorShape({100}); ent->reduce_op = ReduceOp::SUM;
          auto* pp = &ps[i];
          ent->callback = [pp](const Completion& c) { pp->set_value(c.status); };
          std::vector<std::shared_ptr<TensorTableEntry>> es{ent};
          if (!e.EnqueueAllreduces(es, 0).ok()) bad++;
        }
        for (int i = 0; i < 20; ++i) { if (!ps[i].get_future().get().ok()) bad++; if (std::fabs(bufs[i][7] - (float)(n * (n - 1) / 2)) > 1e-4f) bad++; }
      }
      // mismatched shapes -> error on every rank, engine survives
      {
        std::vector<float> v(4 + r, 1.f);
        Status st = run_allreduce("mismatch", v, ReduceOp::SUM);
        if (n > 1 && st.ok()) bad++;
        std::vector<float> w(8, 1.f);
        if (!run_allreduce("after_error", w, ReduceOp::SUM).ok() || std::fabs(w[0] - (float)n) > 1e-5f) bad++;
      }
      // duplicate name while in flight is rejected locally
      {
        // When the first "dup" has already finished, the second is accepted and stays in flight past this scope (it runs
        // once the other ranks send a second "dup" or join), so its callback owns the buffer the engine still reads.
        auto big = std::make_shared<std::vector<float>>(1 << 16, 1.f);
        auto ent = std::make_shared<TensorTableEntry>();
        ent->name = "dup"; ent->input = big->data(); ent->output = big->data(); ent->dtype = DataType::FLOAT32;
        ent->shape = TensorShape({(int64_t)big->size()}); ent->reduce_op = ReduceOp::SUM;
        std::promise<Status> p;
        ent->callback = [&p](const Completion& c) { p.set_value(c.status); };
        std::vector<std::shared_ptr<TensorTableEntry>> es{ent};
        Status st1 = e.EnqueueAllreduces(es, 0);
        auto ent2 = std::make_shared<TensorTableEntry>(*ent);
        ent2->callback = [big](const Completion&) {};
        std::vector<std::shared_ptr<TensorTableEntry>> es2{ent2};
        Status st2 = e.EnqueueAllreduces(es2, 0);
        p.get_future().get();
        if (!st1.ok()) bad++;
        (void)st2;  // may or may not collide depending on timing; must not crash
      }
      // join: rank r does r extra steps first
      {
        for (int s = 0; s < r; ++s) {
          std::vector<float> v(4, 1.f);
          run_allreduce("join." + std::to_string(s), v, ReduceOp::SUM);
        }
        auto ent = std::make_shared<TensorTableEntry>();
        std::promise<int> p;
        ent->callback = [&p](const Completion& c) { p.set_value(c.last_joined_rank); };
        if (!e.EnqueueJoin(ent, 0).ok()) bad++;
        if (p.get_future().get() != n - 1) bad++;
      }
      // process set add / collective inside / remove
      if (n >= 2) {
        std::string err;
        int id = e.AddProcessSet({0, n - 1}, &err);
        if (id <= 0) bad++;
        if (r == 0 || r == n - 1) {
          auto ent = std::make_shared<TensorTableEntry>();
          std::vector<float> v(4, (float)(r + 1));
          ent->name = "ps.t"; ent->input = v.data(); ent->output = v.data(); ent->dtype = DataType::FLOAT32;
          ent->shape = TensorShape({4}); ent->reduce_op = ReduceOp::SUM;
          std::promise<Status> p;
          ent->callback = [&p](const Completion& c) { p.set_value(c.status); };
          std::vector<std::shared_ptr<TensorTableEntry>> es{ent};
          if (!e.EnqueueAllreduces(es, id).ok()) bad++;
          else if (!p.get_future().get().ok() || std::fabs(v[0] - (float)(1 + n)) > 1e-5f) bad++;
        }
        if (e.RemoveProcessSet(id, &err) != id) bad++;
      }
      e.Shutdown();
    });
  }
  for (auto& t : th) t.join();
  CHECK_T(bad.load() == 0);
}

void TestBayes() {
  // maximise -(x-3)^2 - (y+1)^2 on [0,6]x[-4,2]
  BayesianOptimization bo({{0.0, 6.0}, {-4.0, 2.0}}, 0.1);
  std::mt19937 rng(7);
  double best = -1e9;
  for (int i = 0; i < 25; ++i) {
    Vec x = bo.NextSample();
    CHECK_T(x[0] >= 0.0 && x[0] <= 6.0 && x[1] >= -4.0 && x[1] <= 2.0);
    double y = -(x[0] - 3) * (x[0] - 3) - (x[1] + 1) * (x[1] + 1);
    best = std::max(best, y);
    bo.AddSample(x, y);
  }
  CHECK_T(best > -0.6);
  Mat a = {{4, 2}, {2, 3}}, l;
  CHECK_T(Cholesky(a, &l));
  Vec x = CholeskySolve(l, {2, 1});
  CHECK_T(std::fabs(4 * x[0] + 2 * x[1] - 2) < 1e-9 && std::fabs(2 * x[0] + 3 * x[1] - 1) < 1e-9);
}

void TestAutotune() {
  ParameterManager pm;
  pm.Initialize(0, "");
  pm.SetAutoTuning(true);
  int changes = 0;
  for (int i = 0; i < 4000 && pm.IsAutoTuning(); ++i) {
    if (pm.Update({"a", "b"}, 1 << 20)) ++changes;
    if (pm.Update({"a", "b"}, 1 << 20)) ++changes;  // second occurrence of "a" closes a step
  }
  CHECK_T(!pm.IsAutoTuning());
  CHECK_T(changes > 5);
  CHECK_T(pm.params().fusion_threshold_bytes >= (1 << 20));
}
}  // namespace

extern "C" int hvd_selftest(int nranks, char* log, int log_len) {
  g_failures = 0;
  g_log.str("");
  TestWire();
  TestHalf();
  TestFusion();
  TestValidation();
  TestCache();
  TestBayes();
  TestAutotune();
  for (int n : {1, 2, 3, nranks}) { if (n < 1) continue; TestCpuOps(n); TestAdasum(n); }
  for (int n : {2, 3, 5, 6, 7, 8, 11}) TestBitsAmong(n);
  for (int n : {2, 3, 4}) TestShmPlane(n);
  for (int n : {2, 3, 5}) TestTcpMesh(n);
  TestHierPlane(2, 2);
  TestHierPlane(3, 2);
  TestHierPlane(2, 3);
  TestEngines(nranks);
  TestEngines(nranks, 1);
  if (nranks >= 4 && nranks % 2 == 0) TestEngines(nranks, 2);
  TestEngines(1);
  std::string s = g_log.str();
  if (log && log_len > 0) { snprintf(log, log_len, "%s", s.c_str()); }
  return g_failures;
}
