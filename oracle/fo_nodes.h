// ORACLE — TEST INFRASTRUCTURE ONLY (see fo_math.h header). CPU restatement of the *block*
// (`process`) semantics of SamiPerttu/fundsp v0.23.0 for the hot path in SURVEY.md §8a.
// Every class cites the reference file:line it follows. Buffers are [channel][64] f32
// (src/buffer.rs:12-151: channel c, sample i at (c<<6)+i).
#pragma once
#include "fo_math.h"
#include "fo_libm.h"
#include <algorithm>
#include <cassert>
#include <map>
#include <memory>
#include <mutex>
#include <utility>
#include <vector>
#include <xmmintrin.h>

namespace fo {

constexpr int B = MAX_BUFFER_SIZE;
inline int simd_items(int n) { return (n + 7) >> 3; }   // src/lib.rs:76-79
inline int full_simd_items(int n) { return n >> 3; }    // src/lib.rs:82-85

// ---- src/setting.rs:14-62 Parameter / Address / Setting
enum ParamKind { P_NULL = 0, P_CENTER, P_CENTER_Q, P_CENTER_Q_GAIN, P_VALUE, P_COEFFICIENT,
                 P_BIQUAD, P_DELAY, P_TIME, P_ROUGHNESS, P_VARIABILITY, P_PAN,
                 P_ATTACK_RELEASE, P_PHASE, P_SEED, P_INTERVAL };
struct Address { int type; uint64_t value; };  // type 1 = Index, 2 = Node
struct Setting {
  int kind = P_NULL;
  float v[5] = {0, 0, 0, 0, 0};
  uint64_t seed = 0;
  std::vector<Address> address;
  Address direction() const { return address.empty() ? Address{0, 0} : address[0]; }
  Setting peel() const { Setting s = *this; if (!s.address.empty()) s.address.erase(s.address.begin()); return s; }
};

// ---- src/audionode.rs:29-369 AudioNode / src/audiounit.rs:21-95 AudioUnit (merged: oracle is dynamic)
struct Node {
  virtual ~Node() {}
  virtual int inputs() const = 0;
  virtual int outputs() const = 0;
  virtual uint64_t id() const = 0;
  virtual void reset() {}
  virtual void set_sample_rate(double) {}
  virtual void tick(const float* in, float* out) = 0;
  // src/audionode.rs:85-105 default process = per-sample tick.
  virtual void process(int size, const float* in, float* out) {
    float fi[256], fo_[256];
    const int ni = inputs(), no = outputs();
    for (int i = 0; i < size; i++) {
      for (int c = 0; c < ni; c++) fi[c] = in[c * B + i];
      tick(fi, fo_);
      for (int c = 0; c < no; c++) out[c * B + i] = fo_[c];
    }
  }
  // src/audionode.rs:110-126
  void process_remainder(int size, const float* in, float* out) {
    float fi[256], fo_[256];
    const int ni = inputs(), no = outputs();
    for (int i = size & ~7; i < size; i++) {
      for (int c = 0; c < ni; c++) fi[c] = in[c * B + i];
      tick(fi, fo_);
      for (int c = 0; c < no; c++) out[c * B + i] = fo_[c];
    }
  }
  virtual void set(const Setting&) {}
  virtual void set_hash(uint64_t) {}
  // src/audionode.rs:156-161
  virtual AttoHash ping(bool probe, AttoHash hash) {
    if (!probe) { set_hash(hash.state); if (ping_trace()) ping_trace()->push_back(hash.state); }
    return hash.hash(id());
  }
  // test hook: records the hash handed to every leaf during a non-probe ping
  static std::vector<uint64_t>*& ping_trace() { static std::vector<uint64_t>* t = nullptr; return t; }
  virtual Node* clone() const = 0;
  // src/audionode.rs:871-876 etc: constructor-time ping of composite nodes.
  void ctor_ping() { AttoHash h = ping(true, AttoHash(id())); ping(false, h); }
};
typedef std::unique_ptr<Node> NodeP;
#define FO_CLONE(T) Node* clone() const override { return new T(*this); }

// deep-copying child pointer
struct Child {
  NodeP p;
  Child() {}
  explicit Child(Node* n) : p(n) {}
  Child(const Child& o) : p(o.p ? o.p->clone() : nullptr) {}
  Child& operator=(const Child& o) { if (this != &o) p.reset(o.p ? o.p->clone() : nullptr); return *this; }
  Child(Child&& o) noexcept : p(std::move(o.p)) {}
  Child& operator=(Child&& o) noexcept { p = std::move(o.p); return *this; }
  Node* operator->() const { return p.get(); }
};

// ---- src/audionode.rs:374-402 MultiPass (ID 0), :404-433 Pass (ID 48)
struct MultiPass : Node {
  int n; bool single; uint64_t id_override = 0;   // Monitor (ID 56, src/dynamics.rs:441-520) is a pass in the audio path
  MultiPass(int n_, bool single_, uint64_t id_ = 0) : n(n_), single(single_), id_override(id_) {}
  int inputs() const override { return n; } int outputs() const override { return n; }
  uint64_t id() const override { return id_override ? id_override : (single ? 48 : 0); }
  void tick(const float* in, float* out) override { for (int c = 0; c < n; c++) out[c] = in[c]; }
  void process(int size, const float* in, float* out) override {
    for (int c = 0; c < n; c++) for (int i = 0; i < simd_items(size) * 8; i++) out[c * B + i] = in[c * B + i];
  }
  FO_CLONE(MultiPass)
};
// ---- src/audionode.rs:435-465 Sink (ID 1)
struct Sink : Node {
  int n; explicit Sink(int n_) : n(n_) {}
  int inputs() const override { return n; } int outputs() const override { return 0; }
  uint64_t id() const override { return 1; }
  void tick(const float*, float*) override {}
  void process(int, const float*, float*) override {}
  FO_CLONE(Sink)
};
// ---- src/audionode.rs:467-523 Constant (ID 2)
struct Constant : Node {
  std::vector<float> v;
  explicit Constant(std::vector<float> v_) : v(std::move(v_)) {}
  int inputs() const override { return 0; } int outputs() const override { return (int)v.size(); }
  uint64_t id() const override { return 2; }
  void tick(const float*, float* out) override { for (size_t c = 0; c < v.size(); c++) out[c] = v[c]; }
  void process(int size, const float*, float* out) override {
    for (size_t c = 0; c < v.size(); c++) for (int i = 0; i < simd_items(size) * 8; i++) out[c * B + i] = v[c];
  }
  void set(const Setting& s) override { if (s.kind == P_VALUE) for (auto& x : v) x = s.v[0]; }
  FO_CLONE(Constant)
};
// ---- src/audionode.rs:525-567 Split (ID 40), :569-613 MultiSplit (ID 38)
struct MultiSplit : Node {
  int m, n; bool single;
  MultiSplit(int m_, int n_, bool single_) : m(m_), n(n_), single(single_) {}
  int inputs() const override { return m; } int outputs() const override { return m * n; }
  uint64_t id() const override { return single ? 40 : 38; }
  void tick(const float* in, float* out) override { for (int c = 0; c < m * n; c++) out[c] = in[c % m]; }
  void process(int size, const float* in, float* out) override {
    for (int c = 0; c < m * n; c++) for (int i = 0; i < simd_items(size) * 8; i++) out[c * B + i] = in[(c % m) * B + i];
  }
  FO_CLONE(MultiSplit)
};
// ---- src/audionode.rs:615-663 Join (ID 41), :665-722 MultiJoin (ID 39).
// NOTE: tick adds then divides; process scales by z = 1/N then adds (:642-659, :697-718).
struct MultiJoin : Node {
  int m, n; bool single;
  MultiJoin(int m_, int n_, bool single_) : m(m_), n(n_), single(single_) {}
  int inputs() const override { return m * n; } int outputs() const override { return m; }
  uint64_t id() const override { return single ? 41 : 39; }
  void tick(const float* in, float* out) override {
    for (int j = 0; j < m; j++) {
      float o = in[j];
      for (int i = 1; i < n; i++) o += in[j + i * m];
      out[j] = o / (float)(int64_t)n;
    }
  }
  void process(int size, const float* in, float* out) override {
    const float z = 1.0f / (float)(uint64_t)n;
    const int len = simd_items(size) * 8;
    for (int c = 0; c < m; c++) for (int i = 0; i < len; i++) out[c * B + i] = in[c * B + i] * z;
    for (int c = m; c < m * n; c++) for (int i = 0; i < len; i++) out[(c % m) * B + i] += in[c * B + i] * z;
  }
  FO_CLONE(MultiJoin)
};
// ---- src/audionode.rs:2800-2837 Reverse (ID 45)
struct Reverse : Node {
  int n; explicit Reverse(int n_) : n(n_) {}
  int inputs() const override { return n; } int outputs() const override { return n; }
  uint64_t id() const override { return 45; }
  void tick(const float* in, float* out) override { for (int c = 0; c < n; c++) out[c] = in[n - 1 - c]; }
  FO_CLONE(Reverse)
};

// ---- src/audionode.rs:724-1027 Binop (ID 3): x -> temp, y -> out, out = op(temp, out)
enum BinopKind { OP_ADD = 0, OP_SUB = 1, OP_MUL = 2 };
inline float binop(int k, float x, float y) { return k == OP_ADD ? x + y : k == OP_SUB ? x - y : x * y; }
struct Binop : Node {
  int kind; Child x, y; std::vector<float> buf;
  Binop(int k, Node* x_, Node* y_) : kind(k), x(x_), y(y_) {
    assert(x->outputs() == y->outputs());
    buf.assign((size_t)x->outputs() * B, 0.0f);
    ctor_ping();
  }
  int inputs() const override { return x->inputs() + y->inputs(); }
  int outputs() const override { return x->outputs(); }
  uint64_t id() const override { return 3; }
  void reset() override { x->reset(); y->reset(); }
  void set_sample_rate(double sr) override { x->set_sample_rate(sr); y->set_sample_rate(sr); }
  void tick(const float* in, float* out) override {
    float a[256], b[256];
    x->tick(in, a); y->tick(in + x->inputs(), b);
    for (int c = 0; c < outputs(); c++) out[c] = binop(kind, a[c], b[c]);
  }
  void process(int size, const float* in, float* out) override {
    x->process(size, in, buf.data());
    y->process(size, in + x->inputs() * B, out);
    for (int c = 0; c < outputs(); c++)
      for (int i = 0; i < simd_items(size) * 8; i++) out[c * B + i] = binop(kind, buf[c * B + i], out[c * B + i]);
  }
  void set(const Setting& s) override {
    Address d = s.direction();
    if (d.type == 1 && d.value == 0) x->set(s.peel()); else if (d.type == 1 && d.value == 1) y->set(s.peel());
  }
  AttoHash ping(bool probe, AttoHash h) override { return y->ping(probe, x->ping(probe, h.hash(id()))); }
  FO_CLONE(Binop)
};

// ---- src/audionode.rs:1029-1326 Unop (ID 4) with FrameNeg / FrameAddScalar / FrameNegAddScalar / FrameMulScalar
enum UnopKind { U_NEG = 0, U_ADD = 1, U_NEGADD = 2, U_MUL = 3 };
inline float unop(int k, float s, float x) {
  switch (k) { case U_NEG: return -x; case U_ADD: return x + s; case U_NEGADD: return -x + s; default: return x * s; }
}
struct Unop : Node {
  int kind; float scalar; Child x;
  Unop(int k, float s, Node* x_) : kind(k), scalar(s), x(x_) { ctor_ping(); }
  int inputs() const override { return x->inputs(); } int outputs() const override { return x->outputs(); }
  uint64_t id() const override { return 4; }
  void reset() override { x->reset(); }
  void set_sample_rate(double sr) override { x->set_sample_rate(sr); }
  void tick(const float* in, float* out) override {
    x->tick(in, out);
    for (int c = 0; c < outputs(); c++) out[c] = unop(kind, scalar, out[c]);
  }
  void process(int size, const float* in, float* out) override {
    x->process(size, in, out);
    for (int c = 0; c < outputs(); c++) for (int i = 0; i < simd_items(size) * 8; i++) out[c * B + i] = unop(kind, scalar, out[c * B + i]);
  }
  void set(const Setting& s) override { x->set(s); }
  AttoHash ping(bool probe, AttoHash h) override { return x->ping(probe, h.hash(id())); }
  FO_CLONE(Unop)
};

// ---- src/audionode.rs:1370-1492 Pipe (ID 6)
struct Pipe : Node {
  Child x, y; std::vector<float> buf;
  Pipe(Node* x_, Node* y_) : x(x_), y(y_) {
    assert(x->outputs() == y->inputs());
    buf.assign((size_t)std::max(1, x->outputs()) * B, 0.0f);
    ctor_ping();
  }
  int inputs() const override { return x->inputs(); } int outputs() const override { return y->outputs(); }
  uint64_t id() const override { return 6; }
  void reset() override { x->reset(); y->reset(); }
  void set_sample_rate(double sr) override { x->set_sample_rate(sr); y->set_sample_rate(sr); }
  void tick(const float* in, float* out) override { float t[256]; x->tick(in, t); y->tick(t, out); }
  void process(int size, const float* in, float* out) override {
    x->process(size, in, buf.data());
    y->process(size, buf.data(), out);
  }
  void set(const Setting& s) override {
    Address d = s.direction();
    if (d.type == 1 && d.value == 0) x->set(s.peel()); else if (d.type == 1 && d.value == 1) y->set(s.peel());
  }
  AttoHash ping(bool probe, AttoHash h) override { return y->ping(probe, x->ping(probe, h.hash(id()))); }
  FO_CLONE(Pipe)
};

// ---- src/audionode.rs:1494-1649 Stack (ID 7), :1651-1792 Branch (ID 8), :1794-1946 Bus (ID 10)
struct Stack : Node {
  Child x, y;
  Stack(Node* x_, Node* y_) : x(x_), y(y_) { ctor_ping(); }
  int inputs() const override { return x->inputs() + y->inputs(); }
  int outputs() const override { return x->outputs() + y->outputs(); }
  uint64_t id() const override { return 7; }
  void reset() override { x->reset(); y->reset(); }
  void set_sample_rate(double sr) override { x->set_sample_rate(sr); y->set_sample_rate(sr); }
  void tick(const float* in, float* out) override { x->tick(in, out); y->tick(in + x->inputs(), out + x->outputs()); }
  void process(int size, const float* in, float* out) override {
    x->process(size, in, out);
    y->process(size, in + x->inputs() * B, out + x->outputs() * B);
  }
  void set(const Setting& s) override {
    Address d = s.direction();
    if (d.type == 1 && d.value == 0) x->set(s.peel()); else if (d.type == 1 && d.value == 1) y->set(s.peel());
  }
  AttoHash ping(bool probe, AttoHash h) override { return y->ping(probe, x->ping(probe, h.hash(id()))); }
  FO_CLONE(Stack)
};
struct Branch : Node {
  Child x, y;
  Branch(Node* x_, Node* y_) : x(x_), y(y_) { assert(x->inputs() == y->inputs()); ctor_ping(); }
  int inputs() const override { return x->inputs(); }
  int outputs() const override { return x->outputs() + y->outputs(); }
  uint64_t id() const override { return 8; }
  void reset() override { x->reset(); y->reset(); }
  void set_sample_rate(double sr) override { x->set_sample_rate(sr); y->set_sample_rate(sr); }
  void tick(const float* in, float* out) override { x->tick(in, out); y->tick(in, out + x->outputs()); }
  void process(int size, const float* in, float* out) override {
    x->process(size, in, out);
    y->process(size, in, out + x->outputs() * B);
  }
  void set(const Setting& s) override {
    Address d = s.direction();
    if (d.type == 1 && d.value == 0) x->set(s.peel()); else if (d.type == 1 && d.value == 1) y->set(s.peel());
  }
  AttoHash ping(bool probe, AttoHash h) override { return y->ping(probe, x->ping(probe, h.hash(id()))); }
  FO_CLONE(Branch)
};
struct Bus : Node {
  Child x, y; std::vector<float> buf;
  Bus(Node* x_, Node* y_) : x(x_), y(y_) {
    assert(x->inputs() == y->inputs() && x->outputs() == y->outputs());
    buf.assign((size_t)x->outputs() * B, 0.0f);
    ctor_ping();
  }
  int inputs() const override { return x->inputs(); } int outputs() const override { return x->outputs(); }
  uint64_t id() const override { return 10; }
  void reset() override { x->reset(); y->reset(); }
  void set_sample_rate(double sr) override { x->set_sample_rate(sr); y->set_sample_rate(sr); }
  void tick(const float* in, float* out) override {
    float t[256]; x->tick(in, out); y->tick(in, t);
    for (int c = 0; c < outputs(); c++) out[c] = out[c] + t[c];
  }
  void process(int size, const float* in, float* out) override {
    x->process(size, in, out);
    y->process(size, in, buf.data());
    for (int c = 0; c < outputs(); c++) for (int i = 0; i < simd_items(size) * 8; i++) out[c * B + i] += buf[c * B + i];
  }
  void set(const Setting& s) override {
    Address d = s.direction();
    if (d.type == 1 && d.value == 0) x->set(s.peel()); else if (d.type == 1 && d.value == 1) y->set(s.peel());
  }
  AttoHash ping(bool probe, AttoHash h) override { return y->ping(probe, x->ping(probe, h.hash(id()))); }
  FO_CLONE(Bus)
};

// ---- src/audionode.rs:1948-2061 Thru (ID 12): pass missing outputs through from inputs.
struct Thru : Node {
  Child x; std::vector<float> buf;
  explicit Thru(Node* x_) : x(x_) { buf.assign((size_t)std::max(1, x->outputs()) * B, 0.0f); ctor_ping(); }
  int inputs() const override { return x->inputs(); } int outputs() const override { return x->inputs(); }
  uint64_t id() const override { return 12; }
  void reset() override { x->reset(); }
  void set_sample_rate(double sr) override { x->set_sample_rate(sr); }
  void tick(const float* in, float* out) override {
    float t[256]; x->tick(in, t);
    for (int c = 0; c < inputs(); c++) out[c] = c < x->outputs() ? t[c] : in[c];
  }
  void process(int size, const float* in, float* out) override {
    if (x->inputs() == 0) return;
    if (x->outputs() <= x->inputs()) {
      x->process(size, in, out);
    } else {
      x->process(size, in, buf.data());
      for (int c = 0; c < inputs(); c++) for (int i = 0; i < simd_items(size) * 8; i++) out[c * B + i] = buf[c * B + i];
    }
    for (int c = x->outputs(); c < inputs(); c++) for (int i = 0; i < simd_items(size) * 8; i++) out[c * B + i] = in[c * B + i];
  }
  void set(const Setting& s) override { x->set(s); }
  AttoHash ping(bool probe, AttoHash h) override { return x->ping(probe, h.hash(id())); }
  FO_CLONE(Thru)
};

// ---- src/audionode.rs:2063-2200 MultiBus (28), :2202-2355 MultiStack (30), :2357-2530 Reduce (31),
//      :2532-2660 MultiBranch (33), :2662-2800 Chain (32)
enum MultiKind { M_BUS = 28, M_STACK = 30, M_REDUCE = 31, M_BRANCH = 33, M_CHAIN = 32 };
struct Multi : Node {
  int kind; int op; std::vector<Child> x; std::vector<float> buf, buf2;
  Multi(int kind_, int op_, std::vector<Node*> nodes) : kind(kind_), op(op_) {
    for (Node* n : nodes) x.emplace_back(n);
    assert(!x.empty());
    buf.assign((size_t)std::max(1, x[0]->outputs()) * B, 0.0f);
    buf2 = buf;
    ctor_ping();
  }
  int N() const { return (int)x.size(); }
  int inputs() const override {
    switch (kind) { case M_STACK: case M_REDUCE: return x[0]->inputs() * N(); default: return x[0]->inputs(); }
  }
  int outputs() const override {
    switch (kind) { case M_STACK: case M_BRANCH: return x[0]->outputs() * N(); default: return x[0]->outputs(); }
  }
  uint64_t id() const override { return (uint64_t)kind; }
  void reset() override { for (auto& c : x) c->reset(); }
  void set_sample_rate(double sr) override { for (auto& c : x) c->set_sample_rate(sr); }
  void tick(const float* in, float* out) override {
    const int xi = x[0]->inputs(), xo = x[0]->outputs();
    float t[256], u[256];
    switch (kind) {
      case M_BUS:
        x[0]->tick(in, out);
        for (int k = 1; k < N(); k++) { x[k]->tick(in, t); for (int c = 0; c < xo; c++) out[c] = out[c] + t[c]; }
        break;
      case M_STACK: for (int k = 0; k < N(); k++) x[k]->tick(in + k * xi, out + k * xo); break;
      case M_BRANCH: for (int k = 0; k < N(); k++) x[k]->tick(in, out + k * xo); break;
      case M_REDUCE:
        x[0]->tick(in, out);
        for (int k = 1; k < N(); k++) { x[k]->tick(in + k * xi, t); for (int c = 0; c < xo; c++) out[c] = binop(op, out[c], t[c]); }
        break;
      case M_CHAIN:
        for (int c = 0; c < xi; c++) t[c] = in[c];
        for (int k = 0; k < N(); k++) { x[k]->tick(t, u); for (int c = 0; c < xo; c++) t[c] = u[c]; }
        for (int c = 0; c < xo; c++) out[c] = t[c];
        break;
    }
  }
  void process(int size, const float* in, float* out) override {
    const int xi = x[0]->inputs(), xo = x[0]->outputs(), len = simd_items(size) * 8;
    switch (kind) {
      case M_BUS:  // :2124-2135
        x[0]->process(size, in, out);
        for (int k = 1; k < N(); k++) {
          x[k]->process(size, in, buf.data());
          for (int c = 0; c < xo; c++) for (int i = 0; i < len; i++) out[c * B + i] += buf[c * B + i];
        }
        break;
      case M_STACK: for (int k = 0; k < N(); k++) x[k]->process(size, in + k * xi * B, out + k * xo * B); break;
      case M_BRANCH: for (int k = 0; k < N(); k++) x[k]->process(size, in, out + k * xo * B); break;
      case M_REDUCE:  // :2442-2463
        x[0]->process(size, in, out);
        for (int k = 1; k < N(); k++) {
          x[k]->process(size, in + k * xi * B, buf.data());
          for (int c = 0; c < xo; c++) for (int i = 0; i < len; i++) out[c * B + i] = binop(op, out[c * B + i], buf[c * B + i]);
        }
        break;
      case M_CHAIN: {  // :2737-2751 ping-pong
        if (N() == 1) { x[0]->process(size, in, out); break; }
        x[0]->process(size, in, buf.data());
        float* a = buf.data(); float* b = buf2.data();
        for (int k = 1; k < N() - 1; k++) { x[k]->process(size, a, b); std::swap(a, b); }
        x[N() - 1]->process(size, a, out);
        break;
      }
    }
  }
  void set(const Setting& s) override {
    Address d = s.direction();
    if (d.type == 1 && d.value < x.size()) x[d.value]->set(s.peel());
  }
  AttoHash ping(bool probe, AttoHash h) override {
    h = h.hash(id());
    for (auto& c : x) h = c->ping(probe, h);
    return h;
  }
  FO_CLONE(Multi)
};

// ---- src/noise.rs:170-234 Noise (ID 20)
struct Noise : Node {
  uint32_t state = 0; bool has_seed = false; uint64_t seed = 0; uint64_t hash = 0;
  int inputs() const override { return 0; } int outputs() const override { return 1; }
  uint64_t id() const override { return 20; }
  void reset() override { uint64_t h = has_seed ? seed : hash; state = (uint32_t)(h ^ (h >> 32)); }
  void tick(const float*, float* out) override {
    state += 1;
    out[0] = (float)(hash32x(state) >> 8) * (2.0f / (float)((1 << 24) - 1)) - 1.0f;
  }
  void process(int size, const float*, float* out) override {  // :201-215
    const float Z = 2.0f / (float)((1 << 24) - 1);
    for (int i = 0; i < simd_items(size) * 8; i++) out[i] = (float)(hash32x(state + (uint32_t)i + 1u) >> 8) * Z - 1.0f;
    state += (uint32_t)size;
  }
  void set(const Setting& s) override { if (s.kind == P_SEED) { has_seed = true; seed = s.seed; } }
  void set_hash(uint64_t h) override { hash = h; reset(); }
  FO_CLONE(Noise)
};

// ---- src/oscillator.rs:18-102 Sine<f32> (ID 21)
struct Sine : Node {
  float phase = 0, sample_duration = 0; uint64_t hash = 0; bool has_phase = false; float initial_phase = 0;
  Sine() { reset(); set_sample_rate(DEFAULT_SR); }
  int inputs() const override { return 1; } int outputs() const override { return 1; }
  uint64_t id() const override { return 21; }
  void reset() override { phase = has_phase ? initial_phase : (float)rnd1(hash); }
  void set_sample_rate(double sr) override { sample_duration = (float)(1.0 / sr); }
  void tick(const float* in, float* out) override {  // :67-72 (libm::sinf, wrap per sample)
    float p = phase;
    phase += in[0] * sample_duration;
    phase -= floorf(phase);
    out[0] = m::sinf_(p * 6.28318530717958647692f);
  }
  void process(int size, const float* in, float* out) override {  // :74-86 (wide sin, wrap once per block)
    float p = phase;
    for (int i = 0; i < full_simd_items(size); i++) {
      for (int j = 0; j < 8; j++) {
        float tmp = p;
        p += in[(i << 3) + j] * sample_duration;
        out[(i << 3) + j] = wide_sinf(tmp * 6.28318530717958647692f);
      }
    }
    phase = p - floorf(p);
    process_remainder(size, in, out);
  }
  void set(const Setting& s) override { if (s.kind == P_PHASE) { has_phase = true; initial_phase = s.v[0]; } }
  void set_hash(uint64_t h) override { hash = h; reset(); }
  FO_CLONE(Sine)
};

// ---- src/wavetable.rs:24-38 optimal4x44 (T = f32)
inline float optimal4x44(float a0, float a1, float a2, float a3, float x) {
  float z = x - (float)0.5;
  float even1 = a2 + a1, odd1 = a2 - a1, even2 = a3 + a0, odd2 = a3 - a0;
  float c0 = even1 * (float)0.4656725512077848 + even2 * (float)0.03432729708429672;
  float c1 = odd1 * (float)0.5374383075356016 + odd2 * (float)0.1542946255730746;
  float c2 = even1 * (float)-0.25194210134021744 + even2 * (float)0.2519474493593906;
  float c3 = odd1 * (float)-0.46896069955075126 + odd2 * (float)0.15578800670302476;
  float c4 = even1 * (float)0.00986988334359864 + even2 * (float)-0.00989340017126506;
  return (((c4 * z + c3) * z + c2) * z + c1) * z + c0;
}

// ---- src/wavetable.rs:40-242 Wavetable. The inverse FFT (`microfft 0.6.0`, src/fft.rs:51-100, not
// in the reference crate) is replaced by the exact inverse DFT evaluated in f64:
//   x.im[n] * N = sum_k re_k sin(2 pi k n / N) + im_k cos(2 pi k n / N)   (parity unpinned ~1e-7 of peak)
struct Wavetable {
  std::vector<std::pair<float, std::vector<float>>> table;
  static std::vector<float> make_wave(double pitch, double (*phase)(uint32_t), double (*amp)(double, uint32_t)) {
    const double MAX_F = 22000.0, FADE_F = 20000.0;
    size_t harmonics = (size_t)floor(MAX_F / pitch);
    size_t target_len = 4 * harmonics;
    size_t p2 = 1; while (p2 < target_len) p2 <<= 1;
    size_t length = std::min<size_t>(std::max<size_t>(p2, 32), 8192);
    std::vector<double> re(length, 0.0), im(length, 0.0);
    for (size_t i = 1; i <= harmonics; i++) {
      double f = pitch * (double)i;
      double w = amp(pitch, (uint32_t)i);
      w = w * smooth5d(clamp01d(delerpd(MAX_F, FADE_F, f)));
      if (w > 0.0 && i < length) {
        float r = (float)w, th = (float)(6.283185307179586 * phase((uint32_t)i));
        re[i] = (double)(r * cosf(th));  // Complex32::from_polar
        im[i] = (double)(r * sinf(th));
      }
    }
    std::vector<double> sn(length), cs(length);
    for (size_t n = 0; n < length; n++) { sn[n] = sin(6.283185307179586 * (double)n / (double)length); cs[n] = cos(6.283185307179586 * (double)n / (double)length); }
    std::vector<float> out(length);
    for (size_t n = 0; n < length; n++) {
      double acc = 0.0;
      for (size_t k = 1; k <= harmonics && k < length; k++) {
        size_t a = (k * n) & (length - 1);
        acc += re[k] * sn[a] + im[k] * cs[a];
      }
      out[n] = (float)acc;
    }
    return out;
  }
  Wavetable(double min_pitch, double max_pitch, double tables_per_octave, double (*phase)(uint32_t), double (*amp)(double, uint32_t)) {
    double pitch = min_pitch;
    double p_factor = pow(2.0, 1.0 / tables_per_octave);
    float max_amplitude = 0.0f;
    while (pitch <= max_pitch) {
      std::vector<float> wave = make_wave(pitch, phase, amp);
      for (float x : wave) max_amplitude = fmaxf(max_amplitude, fabsf(x));
      table.emplace_back((float)pitch, std::move(wave));
      pitch *= p_factor;
    }
    if (max_amplitude > 0.0f) {
      float z = 1.0f / max_amplitude;
      for (auto& t : table) for (float& x : t.second) x *= z;
    }
  }
  float at(size_t i, float phase) const {  // :125-137
    const std::vector<float>& t = table[i].second;
    float p = (float)t.size() * phase;
    size_t i1 = (size_t)p;
    float w = p - (float)i1;
    size_t mask = t.size() - 1;
    size_t i0 = (i1 - 1) & mask; i1 &= mask;
    size_t i2 = (i1 + 1) & mask, i3 = (i1 + 2) & mask;
    return optimal4x44(t[i0], t[i1], t[i2], t[i3], w);
  }
  float at_simd_lane(size_t i, float phase) const {  // :139-155 (i32 lanes, fast_trunc_int)
    const std::vector<float>& t = table[i].second;
    float p = (float)t.size() * phase;
    int32_t i1 = (int32_t)p;  // cvttps2dq: truncation toward zero
    float w = p - (float)i1;
    int32_t mask = (int32_t)t.size() - 1;
    int32_t i0 = (i1 - 1) & mask; i1 &= mask;
    int32_t i2 = (i1 + 1) & mask, i3 = (i2 + 1) & mask;
    return optimal4x44(t[i0], t[i1], t[i2], t[i3], w);
  }
  size_t table_index(size_t hint, float frequency) const {  // :157-179
    if (frequency >= table[hint].first && frequency <= table[hint + 1].first) return hint;
    size_t i0 = 0, i1 = table.size() - 3;
    while (i0 < i1) {
      size_t i = (i0 + i1) >> 1;
      if (table[i].first > frequency) i1 = i;
      else if (table[i + 1].first > frequency) { i0 = i; break; }
      else i0 = i + 1;
    }
    return i0;
  }
};

inline double ph_saw(uint32_t i) { return (i & 1) == 1 ? 0.0 : 0.5; }
inline double am_saw(double, uint32_t i) { return 1.0 / (double)i; }
inline double ph_zero(uint32_t) { return 0.0; }
inline double am_square(double, uint32_t i) { return (i & 1) == 1 ? 1.0 / (double)i : 0.0; }
inline double ph_tri(uint32_t i) { return (i & 3) == 3 ? 0.5 : 0.0; }
inline double am_tri(double, uint32_t i) { return (i & 1) == 1 ? 1.0 / (double)(i * i) : 0.0; }
inline double ph_organ(uint32_t i) { return (i & 3) == 3 ? 0.5 : ((i & 1) == 1 ? 0.0 : 0.5); }
inline double am_organ(double, uint32_t i) { uint32_t z = __builtin_ctz(i); uint32_t j = i >> z; return 1.0 / (double)(i + j * j * j); }
inline double am_softsaw(double, uint32_t i) { return 1.0 / (double)(i * i); }
inline double am_hammond(double, uint32_t i) {
  uint32_t z = __builtin_ctz(i); uint32_t j = i >> z; double f = 1.0 / (double)((z + 1) * (z + 1));
  if (i == 1 || i == 2 || i == 3) return 1.0;
  if (j == 1 || j == 3) return f;
  if (j == 9) return 0.2 * f;
  return 0.0;
}
// ---- src/wavetable.rs:493-623 global tables: 0 saw, 1 square, 2 triangle, 3 organ, 4 soft_saw, 5 hammond
inline const Wavetable& global_table(int kind) {
  static std::unique_ptr<Wavetable> t[6];
  static std::once_flag once[6];   // the bank renderer calls this from worker threads: build each table exactly once
  std::call_once(once[kind], [kind]() {
    switch (kind) {
      case 0: t[0].reset(new Wavetable(20.0, 20000.0, 4.0, ph_saw, am_saw)); break;
      case 1: t[1].reset(new Wavetable(20.0, 20000.0, 4.0, ph_zero, am_square)); break;
      case 2: t[2].reset(new Wavetable(20.0, 20000.0, 4.0, ph_tri, am_tri)); break;
      case 3: t[3].reset(new Wavetable(20.0, 20000.0, 4.0, ph_organ, am_organ)); break;
      case 4: t[4].reset(new Wavetable(20.0, 20000.0, 4.0, ph_organ, am_softsaw)); break;
      default: t[5].reset(new Wavetable(20.0, 20000.0, 4.0, ph_zero, am_hammond)); break;
    }
  });
  return *t[kind];
}

// ---- src/wavetable.rs:244-359 WaveSynth<N> (ID 34)
struct WaveSynth : Node {
  int kind, nout; float phase = 0; uint64_t hash = 0; bool has_phase = false; float initial_phase = 0;
  size_t table_hint = 0; float sample_rate = (float)DEFAULT_SR; float sample_duration = 1.0f / (float)DEFAULT_SR;
  WaveSynth(int kind_, int nout_) : kind(kind_), nout(nout_) {}
  const Wavetable& tab() const { return global_table(kind); }
  int inputs() const override { return 1; } int outputs() const override { return nout; }
  uint64_t id() const override { return 34; }
  void reset() override { phase = has_phase ? initial_phase : (float)rnd1(hash); }
  void set_sample_rate(double sr) override { sample_rate = (float)sr; sample_duration = 1.0f / (float)sr; }
  void set_hash(uint64_t h) override { hash = h; reset(); }
  void tick(const float* in, float* out) override {  // :309-325
    float frequency = in[0];
    phase += frequency * sample_duration;
    phase -= floorf(phase);
    const Wavetable& t = tab();
    size_t ti = t.table_index(table_hint, fabsf(frequency));
    float w = clamp01f(delerpf(t.table[ti].first, t.table[ti + 1].first, fabsf(frequency)));
    float o = (1.0f - w) * t.at(ti + 1, phase) + w * t.at(ti + 2, phase);
    table_hint = ti;
    out[0] = o; if (nout > 1) out[1] = phase;
  }
  void process(int size, const float* in, float* out) override {  // :327-348
    float p = phase; size_t hint = table_hint; const Wavetable& t = tab();
    for (int i = 0; i < full_simd_items(size); i++) {
      float frequency = in[i << 3];
      float ph[8];
      for (int j = 0; j < 8; j++) { p += in[(i << 3) + j] * sample_duration; ph[j] = p; }
      for (int j = 0; j < 8; j++) ph[j] = ph[j] - wide_floorf(ph[j]);
      size_t ti = t.table_index(hint, fabsf(frequency));
      float w = clamp01f(delerpf(t.table[ti].first, t.table[ti + 1].first, fabsf(frequency)));
      for (int j = 0; j < 8; j++) {
        out[(i << 3) + j] = (1.0f - w) * t.at_simd_lane(ti + 1, ph[j]) + w * t.at_simd_lane(ti + 2, ph[j]);
        if (nout > 1) out[B + (i << 3) + j] = ph[j];
      }
      hint = ti;
    }
    phase = p - floorf(p);
    table_hint = hint;
    process_remainder(size, in, out);
  }
  void set(const Setting& s) override { if (s.kind == P_PHASE) { has_phase = true; initial_phase = s.v[0]; } }
  FO_CLONE(WaveSynth)
};

// ---- src/wavetable.rs:361-433 PhaseSynth (ID 35): table lookup at an input phase; no block override (default process = tick)
struct PhaseSynth : Node {
  int kind; float phase = 0; bool phase_ready = false; size_t table_hint = 0; float sample_rate = (float)DEFAULT_SR;
  explicit PhaseSynth(int k) : kind(k) {}
  int inputs() const override { return 1; } int outputs() const override { return 1; }
  uint64_t id() const override { return 35; }
  void reset() override { phase_ready = false; }
  void set_sample_rate(double sr) override { sample_rate = (float)sr; }
  void tick(const float* in, float* out) override {  // :400-428
    float ph = in[0]; ph = ph - floorf(ph);
    float delta;
    if (phase_ready) delta = fminf(fabsf(ph - phase), fminf(fabsf(ph - 1.0f - phase), fabsf(ph + 1.0f - phase)));
    else { phase_ready = true; delta = 0.5f; }
    const Wavetable& t = global_table(kind);
    const float frequency = delta * sample_rate;
    size_t ti = t.table_index(table_hint, frequency);   // Wavetable::read :181-195
    float w = clamp01f(delerpf(t.table[ti].first, t.table[ti + 1].first, frequency));
    out[0] = (1.0f - w) * t.at(ti + 1, ph) + w * t.at(ti + 2, ph);
    table_hint = ti; phase = ph;
  }
  FO_CLONE(PhaseSynth)
};
// ---- src/wavetable.rs:439-491 PulseWave (ID 44): difference of two saws, the second read at phase + width
struct PulseWave : Node {
  Child pulse;
  PulseWave() {
    Node* a = new Stack(new WaveSynth(0, 2), new MultiPass(1, true));
    Node* b = new Stack(new MultiPass(1, true), new Pipe(new Binop(0, new MultiPass(1, true), new MultiPass(1, true)), new PhaseSynth(0)));
    pulse = Child(new Pipe(new Pipe(a, b), new Binop(1, new MultiPass(1, true), new MultiPass(1, true))));
  }
  int inputs() const override { return 2; } int outputs() const override { return 1; }
  uint64_t id() const override { return 44; }
  void reset() override { pulse->reset(); }
  void set_sample_rate(double sr) override { pulse->set_sample_rate(sr); }
  void tick(const float* in, float* out) override { pulse->tick(in, out); }
  void process(int size, const float* in, float* out) override { pulse->process(size, in, out); }
  void set(const Setting& s) override {   // :479-481 left_mut().left_mut().left_mut()
    Setting t = s; t.address.insert(t.address.begin(), {Address{1, 0}, Address{1, 0}, Address{1, 0}}); pulse->set(t);
  }
  AttoHash ping(bool probe, AttoHash h) override { return pulse->ping(probe, h).hash(id()); }
  FO_CLONE(PulseWave)
};

// ---- src/svf.rs:16-221 SvfCoefs<f32>; modes 0 lowpass 1 highpass 2 bandpass 3 notch 4 peak 5 allpass 6 bell 7 lowshelf 8 highshelf
struct SvfCoefs { float a1 = 0, a2 = 0, a3 = 0, m0 = 0, m1 = 0, m2 = 0; };
inline SvfCoefs svf_coefs(int mode, float sr, float cutoff, float q, float gain) {
  const float PI_F = (float)3.14159265358979323846;
  SvfCoefs c; float g, k;
  if (mode <= 5) {
    g = m::tanf_(PI_F * cutoff / sr); k = 1.0f / q;
  } else if (mode == 6) {
    float a = sqrtf(gain); g = m::tanf_(PI_F * cutoff / sr); k = 1.0f / (q * a);
    c.m0 = 1.0f; c.m1 = k * (a * a - 1.0f); c.m2 = 0.0f;
  } else if (mode == 7) {
    float a = sqrtf(gain); g = m::tanf_(PI_F * cutoff / sr) / sqrtf(a); k = 1.0f / q;
    c.m0 = 1.0f; c.m1 = k * (a - 1.0f); c.m2 = a * a - 1.0f;
  } else {
    float a = sqrtf(gain); g = m::tanf_(PI_F * cutoff / sr) * sqrtf(a); k = 1.0f / q;
    c.m0 = a * a; c.m1 = k * (1.0f - a) * a; c.m2 = 1.0f - a * a;
  }
  c.a1 = 1.0f / (1.0f + g * (g + k)); c.a2 = g * c.a1; c.a3 = g * c.a2;
  switch (mode) {
    case 0: c.m0 = 0.0f; c.m1 = 0.0f; c.m2 = 1.0f; break;
    case 1: c.m0 = 1.0f; c.m1 = -k; c.m2 = -1.0f; break;
    case 2: c.m0 = 0.0f; c.m1 = 1.0f; c.m2 = 0.0f; break;
    case 3: c.m0 = 1.0f; c.m1 = -k; c.m2 = 0.0f; break;
    case 4: c.m0 = 1.0f; c.m1 = -k; c.m2 = -2.0f; break;
    case 5: c.m0 = 1.0f; c.m1 = -2.0f * k; c.m2 = 0.0f; break;
    default: break;
  }
  return c;
}
// ---- src/svf.rs:744-855 Svf (ID 36, parameter inputs) and :857-1031 FixedSvf (ID 43)
struct Svf : Node {
  int mode; bool fixed; float sr, cutoff, q, gain; SvfCoefs c; float ic1eq = 0, ic2eq = 0;
  Svf(int mode_, bool fixed_, float cutoff_, float q_, float gain_) : mode(mode_), fixed(fixed_), sr((float)DEFAULT_SR), cutoff(cutoff_), q(q_), gain(gain_) { update(); }
  void update() { c = svf_coefs(mode, sr, cutoff, q, gain); }
  int inputs() const override { return fixed ? 1 : (mode >= 6 ? 4 : 3); } int outputs() const override { return 1; }
  uint64_t id() const override { return fixed ? 43 : 36; }
  void reset() override { ic1eq = 0; ic2eq = 0; }
  void set_sample_rate(double s) override { sr = (float)s; update(); }
  void tick(const float* in, float* out) override {
    if (!fixed) {  // update_inputs (svf.rs:305-312 etc.): recompute only on change
      if (mode >= 6) { if (in[1] != cutoff || in[2] != q || in[3] != gain) { cutoff = in[1]; q = in[2]; gain = in[3]; update(); } }
      else if (in[1] != cutoff || in[2] != q) { cutoff = in[1]; q = in[2]; update(); }
    }
    float v0 = in[0];
    float v3 = v0 - ic2eq;
    float v1 = c.a1 * ic1eq + c.a2 * v3;
    float v2 = ic2eq + c.a2 * ic1eq + c.a3 * v3;
    ic1eq = 2.0f * v1 - ic1eq;
    ic2eq = 2.0f * v2 - ic2eq;
    out[0] = c.m0 * v0 + c.m1 * v1 + c.m2 * v2;
  }
  void set(const Setting& s) override {
    if (!fixed) return;
    if (s.kind == P_CENTER) { cutoff = s.v[0]; update(); }
    else if (s.kind == P_CENTER_Q) { cutoff = s.v[0]; q = s.v[1]; update(); }
    else if (s.kind == P_CENTER_Q_GAIN) { cutoff = s.v[0]; q = s.v[1]; gain = s.v[2]; update(); }
  }
  FO_CLONE(Svf)
};

// ---- src/svf.rs:1034-1111 Morph (ID 62): peak SVF morphing between lowpass, peak and highpass; inputs (audio, cutoff, q, morph)
struct Morph : Node {
  Svf filter;
  Morph(float cutoff, float q) : filter(4 /* PeakMode */, false, cutoff, q, 0.0f) { ctor_ping(); }
  int inputs() const override { return 4; } int outputs() const override { return 1; }
  uint64_t id() const override { return 62; }
  void reset() override { filter.reset(); }
  void set_sample_rate(double s) override { filter.set_sample_rate(s); }
  void tick(const float* in, float* out) override { float y; filter.tick(in, &y); out[0] = (y + in[3] * in[0]) * 0.5f; }
  AttoHash ping(bool probe, AttoHash h) override { return filter.ping(probe, h).hash(id()); }   // :1108-1110 (filter first, then the ID)
  FO_CLONE(Morph)
};
// ---- src/rez.rs Rez<F, N> (ID 75, F = f32): Paul Kellett's resonant two-pole; bandpass = 0 lowrez, 1 bandrez
struct Rez : Node {
  int nin; float bandpass, cutoff, q, f = 1, fb = 1, sr = (float)DEFAULT_SR, buf0 = 0, buf1 = 0;
  Rez(float bandpass_, float cutoff_, float q_, int nin_) : nin(nin_), bandpass(bandpass_), cutoff(cutoff_), q(q_) { set_cutoff_q(cutoff_, q_); }
  void set_cutoff_q(float c, float qq) {
    cutoff = c; f = 2.0f * m::sinf_(3.14159274101257324f * c / sr);
    q = qq; fb = qq + qq / (1.0f - f);
  }
  int inputs() const override { return nin; } int outputs() const override { return 1; }
  uint64_t id() const override { return 75; }
  void reset() override { buf0 = buf1 = 0; }
  void set_sample_rate(double s) override { sr = (float)s; set_cutoff_q(cutoff, q); }
  void tick(const float* in, float* out) override {
    if (nin > 1 && (in[1] != cutoff || in[2] != q)) set_cutoff_q(in[1], in[2]);
    const float hp = in[0] - buf0, bp = buf0 - buf1;
    buf0 += f * (hp + fb * m::tanhf_(bp));
    buf1 += f * (buf0 - buf1);
    out[0] = buf1 - bandpass * buf0;
  }
  void set(const Setting& s) override {
    if (s.kind == P_CENTER) set_cutoff_q(s.v[0], q);
    else if (s.kind == P_CENTER_Q) set_cutoff_q(s.v[0], s.v[1]);
  }
  FO_CLONE(Rez)
};

// ---- src/biquad.rs:17-116 BiquadCoefs<f32>
struct BiquadCoefs { float a1 = 0, a2 = 0, b0 = 0, b1 = 0, b2 = 0; };
inline BiquadCoefs biquad_butter_lowpass(float sr, float cutoff) {
  const float PI_F = 3.14159274101257324f, SQRT_2 = 1.41421354f;
  float f = m::tanf_(cutoff * PI_F / sr);
  float a0r = 1.0f / (1.0f + SQRT_2 * f + f * f);
  BiquadCoefs c; c.a1 = (2.0f * f * f - 2.0f) * a0r; c.a2 = (1.0f - SQRT_2 * f + f * f) * a0r;
  c.b0 = f * f * a0r; c.b1 = 2.0f * c.b0; c.b2 = c.b0; return c;
}
inline BiquadCoefs biquad_resonator(float sr, float center, float q) {
  const float PI_F = 3.14159274101257324f, TAU_F = 6.28318548202514648f;
  float r = m::expf_(-PI_F * center / (q * sr));
  BiquadCoefs c; c.a1 = -2.0f * r * m::cosf_(TAU_F * center / sr); c.a2 = r * r;
  c.b0 = sqrtf(1.0f - r * r) * 0.5f; c.b1 = 0.0f; c.b2 = -c.b0; return c;
}
inline BiquadCoefs biquad_lowpass(float sr, float cutoff, float q) {
  const float TAU_F = 6.28318548202514648f;
  float omega = TAU_F * cutoff / sr;
  float alpha = m::sinf_(omega) / (2.0f * q);
  float beta = m::cosf_(omega);
  float a0r = 1.0f / (1.0f + alpha);
  BiquadCoefs c; c.a1 = -2.0f * beta * a0r; c.a2 = (1.0f - alpha) * a0r;
  c.b1 = (1.0f - beta) * a0r; c.b0 = c.b1 * 0.5f; c.b2 = c.b0; return c;
}
inline BiquadCoefs biquad_highpass(float sr, float cutoff, float q) {
  const float TAU_F = 6.28318548202514648f;
  float omega = TAU_F * cutoff / sr;
  float alpha = m::sinf_(omega) / (2.0f * q);
  float beta = m::cosf_(omega);
  float a0r = 1.0f / (1.0f + alpha);
  BiquadCoefs c; c.a1 = -2.0f * beta * a0r; c.a2 = (1.0f - alpha) * a0r;
  c.b0 = (1.0f + beta) * 0.5f * a0r; c.b1 = (-1.0f - beta) * a0r; c.b2 = c.b0; return c;
}
inline BiquadCoefs biquad_bell(float sr, float center, float q, float gain) {
  const float TAU_F = 6.28318548202514648f;
  float omega = TAU_F * center / sr;
  float alpha = m::sinf_(omega) / (2.0f * q);
  float beta = m::cosf_(omega);
  float a = sqrtf(gain);
  float a0r = 1.0f / (1.0f + alpha / a);
  BiquadCoefs c; c.a1 = -2.0f * beta * a0r; c.a2 = (1.0f - alpha / a) * a0r;
  c.b0 = (1.0f + alpha * a) * a0r; c.b1 = c.a1; c.b2 = (1.0f - alpha * a) * a0r; return c;
}
// ---- src/biquad.rs:130-218 Biquad<f32> (ID 15): DF1, evaluated left to right.
struct Biquad : Node {
  BiquadCoefs c; float x1 = 0, x2 = 0, y1 = 0, y2 = 0;
  explicit Biquad(BiquadCoefs c_) : c(c_) {}
  int inputs() const override { return 1; } int outputs() const override { return 1; }
  uint64_t id() const override { return 15; }
  void reset() override { x1 = x2 = y1 = y2 = 0; }
  void tick(const float* in, float* out) override {
    float x0 = in[0];
    float y0 = c.b0 * x0 + c.b1 * x1 + c.b2 * x2 - c.a1 * y1 - c.a2 * y2;
    x2 = x1; x1 = x0; y2 = y1; y1 = y0; out[0] = y0;
  }
  void set(const Setting& s) override { if (s.kind == P_BIQUAD) { c.a1 = s.v[0]; c.a2 = s.v[1]; c.b0 = s.v[2]; c.b1 = s.v[3]; c.b2 = s.v[4]; } }
  FO_CLONE(Biquad)
};
// ---- src/biquad.rs:220-299 ButterLowpass<f32,N> (ID 16), :301-382 Resonator<f32,N> (ID 17)
struct ButterLowpass : Node {
  int nin; Biquad bq; float sr, cutoff;
  ButterLowpass(float cutoff_, int nin_) : nin(nin_), bq(BiquadCoefs()), sr((float)DEFAULT_SR), cutoff(0) { set_cutoff(cutoff_); }
  void set_cutoff(float c) { bq.c = biquad_butter_lowpass(sr, c); cutoff = c; }
  int inputs() const override { return nin; } int outputs() const override { return 1; }
  uint64_t id() const override { return 16; }
  void reset() override { bq.reset(); }
  void set_sample_rate(double s) override { sr = (float)s; bq.set_sample_rate(s); set_cutoff(cutoff); }
  void tick(const float* in, float* out) override {
    if (nin > 1) { float c = in[1]; if (c != cutoff) set_cutoff(c); }
    bq.tick(in, out);
  }
  void set(const Setting& s) override { if (s.kind == P_CENTER) set_cutoff(s.v[0]); }
  FO_CLONE(ButterLowpass)
};
struct Resonator : Node {
  int nin; Biquad bq; float sr, center, q;
  Resonator(float center_, float q_, int nin_) : nin(nin_), bq(BiquadCoefs()), sr((float)DEFAULT_SR), center(0), q(0) { set_center_q(center_, q_); }
  void set_center_q(float c, float q_) { bq.c = biquad_resonator(sr, c, q_); center = c; q = q_; }
  int inputs() const override { return nin; } int outputs() const override { return 1; }
  uint64_t id() const override { return 17; }
  void reset() override { bq.reset(); }
  void set_sample_rate(double s) override { sr = (float)s; set_center_q(center, q); }
  void tick(const float* in, float* out) override {
    if (nin >= 3) { float c = in[1], qq = in[2]; if (c != center || qq != q) set_center_q(c, qq); }
    bq.tick(in, out);
  }
  void set(const Setting& s) override { if (s.kind == P_CENTER) set_center_q(s.v[0], q); else if (s.kind == P_CENTER_Q) set_center_q(s.v[0], s.v[1]); }
  FO_CLONE(Resonator)
};
// ---- src/biquad_bank.rs:9-117 BiquadBank<f32x8> (ID 98): 8 lanes, one per channel.
struct BiquadBank : Node {
  BiquadCoefs c[8]; float x1[8] = {0}, x2[8] = {0}, y1[8] = {0}, y2[8] = {0};
  int inputs() const override { return 8; } int outputs() const override { return 8; }
  uint64_t id() const override { return 98; }
  void reset() override { for (int l = 0; l < 8; l++) x1[l] = x2[l] = y1[l] = y2[l] = 0; }
  void tick(const float* in, float* out) override {
    for (int l = 0; l < 8; l++) {
      float x0 = in[l];
      float y0 = c[l].b0 * x0 + c[l].b1 * x1[l] + c[l].b2 * x2[l] - c[l].a1 * y1[l] - c[l].a2 * y2[l];
      x2[l] = x1[l]; x1[l] = x0; y2[l] = y1[l]; y1[l] = y0; out[l] = y0;
    }
  }
  void set(const Setting& s) override {
    Address d = s.direction();
    if (d.type == 1 && s.kind == P_BIQUAD && d.value < 8) { BiquadCoefs& k = c[d.value]; k.a1 = s.v[0]; k.a2 = s.v[1]; k.b0 = s.v[2]; k.b1 = s.v[3]; k.b2 = s.v[4]; }
  }
  FO_CLONE(BiquadBank)
};

// ---- src/moog.rs:11-117 Moog<f32, N> (ID 60)
struct Moog : Node {
  int nin; float q = 0, cutoff = 0, sr, rez = 0, p = 0, k = 0, s0 = 0, s1 = 0, s2 = 0, s3 = 0, px = 0, ps0 = 0, ps1 = 0, ps2 = 0;
  Moog(float cutoff_, float q_, int nin_) : nin(nin_), sr((float)DEFAULT_SR) { set_cutoff_q(cutoff_, q_); }
  void set_cutoff_q(float cutoff_, float q_) {  // :48-57
    cutoff = cutoff_; q = q_;
    float c = 2.0f * cutoff / sr;
    p = c * (1.8f - 0.8f * c);
    k = 2.0f * m::sinf_(c * 3.14159274101257324f * 0.5f) - 1.0f;
    float t1 = (1.0f - p) * 1.386249f;
    float t2 = 12.0f + t1 * t1;
    rez = q * (t2 + 6.0f * t1) / (t2 - 6.0f * t1);
  }
  int inputs() const override { return nin; } int outputs() const override { return 1; }
  uint64_t id() const override { return 60; }
  void reset() override { s0 = s1 = s2 = s3 = px = ps0 = ps1 = ps2 = 0; }
  void set_sample_rate(double s) override { sr = (float)s; set_cutoff_q(cutoff, q); }
  void tick(const float* in, float* out) override {  // :81-100
    if (nin > 1) set_cutoff_q(in[1], in[2]);
    float x = -rez * s3 + in[0];
    s0 = (x + px) * p - k * s0;
    s1 = (s0 + ps0) * p - k * s1;
    s2 = (s1 + ps1) * p - k * s2;
    s3 = m::tanhf_((s2 + ps2) * p - k * s3);
    px = x; ps0 = s0; ps1 = s1; ps2 = s2;
    out[0] = s3;
  }
  void set(const Setting& s) override { if (s.kind == P_CENTER) set_cutoff_q(s.v[0], q); else if (s.kind == P_CENTER_Q) set_cutoff_q(s.v[0], s.v[1]); }
  FO_CLONE(Moog)
};

// ---- src/fir.rs:11-89 Fir<N> (ID 52)
struct Fir : Node {
  std::vector<float> w, v;
  explicit Fir(std::vector<float> w_) : w(std::move(w_)), v(w.size(), 0.0f) {}
  int inputs() const override { return 1; } int outputs() const override { return 1; }
  uint64_t id() const override { return 52; }
  void reset() override { std::fill(v.begin(), v.end(), 0.0f); }
  void tick(const float* in, float* out) override {
    const size_t n = w.size();
    for (size_t i = 0; i + 1 < n; i++) v[i] = v[i + 1];
    v[n - 1] = in[0];
    float o = 0.0f;
    for (size_t i = 0; i < n; i++) o += w[i] * v[i];
    out[0] = o;
  }
  FO_CLONE(Fir)
};

// ---- src/delay.rs:17-65 Tick<N> (ID 9)
struct TickNode : Node {
  std::vector<float> buf; explicit TickNode(int n) : buf(n, 0.0f) {}
  int inputs() const override { return (int)buf.size(); } int outputs() const override { return (int)buf.size(); }
  uint64_t id() const override { return 9; }
  void reset() override { std::fill(buf.begin(), buf.end(), 0.0f); }
  void tick(const float* in, float* out) override { for (size_t c = 0; c < buf.size(); c++) { float t = buf[c]; buf[c] = in[c]; out[c] = t; } }
  FO_CLONE(TickNode)
};
// ---- src/delay.rs:67-139 Delay (ID 13)
struct Delay : Node {
  std::vector<float> buffer; size_t i = 0; double sample_rate = 0.0, time; size_t time_in_samples = 0;
  explicit Delay(double t) : time(t) { assert(t >= 0.0); set_sample_rate(DEFAULT_SR); }
  int inputs() const override { return 1; } int outputs() const override { return 1; }
  uint64_t id() const override { return 13; }
  void reset() override { i = 0; std::fill(buffer.begin(), buffer.end(), 0.0f); }
  void set_sample_rate(double sr) override {
    if (sample_rate != sr) {
      sample_rate = sr;
      time_in_samples = (size_t)round(time * sr);
      buffer.resize(time_in_samples + 1, 0.0f);
      reset();
    }
  }
  void tick(const float* in, float* out) override {
    buffer[i] = in[0];
    i += 1; if (i >= buffer.size()) i = 0;
    out[0] = buffer[i];
  }
  FO_CLONE(Delay)
};
// ---- src/delay.rs:288-377 AllNest<N,X> (ID 83)
struct AllNest : Node {
  int nin; Child x; float eta, z = 0;
  AllNest(float coefficient, Node* x_, int nin_) : nin(nin_), x(x_), eta(coefficient) {}
  int inputs() const override { return nin; } int outputs() const override { return 1; }
  uint64_t id() const override { return 83; }
  void reset() override { z = 0; x->reset(); }
  void set_sample_rate(double sr) override { x->set_sample_rate(sr); }
  void tick(const float* in, float* out) override {
    if (nin > 1) eta = in[1];
    float v = in[0] - eta * z;
    float y = eta * v + z;
    float o; x->tick(&v, &o); z = o;
    out[0] = y;
  }
  void set(const Setting& s) override { if (s.kind == P_COEFFICIENT) eta = s.v[0]; }
  AttoHash ping(bool probe, AttoHash h) override { return x->ping(probe, h.hash(id())); }
  FO_CLONE(AllNest)
};

// ---- src/reverb.rs:139-279 Reverb<F> (ID 85): allpass-loop stereo reverb with a user loop filter (reverb3_stereo)
struct Reverb85 : Node {
  struct Block { std::unique_ptr<Node> delay, ap0[4], ap1[4], f0, f1; };
  std::unique_ptr<Node> pre[4]; Block block[8]; float feedback = 0, a;
  static Node* schroeder(float coeff, int samples) { return new AllNest(coeff, new Delay((double)(samples - 1) / DEFAULT_SR), 1); }
  Reverb85(double time, double diffusion, Node* filter) {   // :156-206 (takes ownership of `filter`, clones it per loop position)
    static const int ldelays[32] = {401, 421, 443, 463, 487, 503, 523, 547, 563, 587, 607, 619, 643, 661, 683, 701, 727, 743, 761, 787, 809, 823, 839, 863, 883, 907, 929, 947, 967, 983, 1009, 1021};
    static const int rdelays[32] = {419, 433, 457, 479, 491, 509, 541, 557, 577, 593, 613, 631, 653, 673, 691, 719, 733, 757, 773, 797, 811, 829, 853, 877, 887, 911, 937, 953, 977, 997, 1013, 1033};
    static const int delays[8] = {1087, 1091, 1093, 1097, 1103, 1109, 1117, 1123};
    static const int predelay[4] = {245, 367, 263, 349};
    const float coeff = (float)(0.5 * (1.0 - diffusion) + 0.9 * diffusion);   // lerp(0.5, 0.9, diffusion) = a*(1-t) + b*t
    for (int i = 0; i < 8; i++) {
      for (int j = 0; j < 4; j++) { block[i].ap0[j].reset(schroeder(coeff, ldelays[i + j * 8])); block[i].ap1[j].reset(schroeder(coeff, rdelays[i + j * 8])); }
      block[i].delay.reset(new Delay((double)delays[7 - i] / DEFAULT_SR));
      block[i].f0.reset(filter->clone()); block[i].f1.reset(filter->clone());
    }
    a = (float)pow(db_ampd(-60.0), 0.035 / time);                               // pow(db_amp(-60.0), 0.035 / time) as f32
    for (int i = 0; i < 4; i++) pre[i].reset(schroeder(coeff, predelay[i]));
    delete filter;
  }
  Reverb85(const Reverb85& o) : Node(o), feedback(o.feedback), a(o.a) {
    for (int i = 0; i < 4; i++) pre[i].reset(o.pre[i]->clone());
    for (int i = 0; i < 8; i++) {
      for (int j = 0; j < 4; j++) { block[i].ap0[j].reset(o.block[i].ap0[j]->clone()); block[i].ap1[j].reset(o.block[i].ap1[j]->clone()); }
      block[i].delay.reset(o.block[i].delay->clone()); block[i].f0.reset(o.block[i].f0->clone()); block[i].f1.reset(o.block[i].f1->clone());
    }
  }
  int inputs() const override { return 2; } int outputs() const override { return 2; }
  uint64_t id() const override { return 85; }
  template <class Fn> void each(Fn fn) {
    for (auto& b : block) { for (auto& x : b.ap0) fn(*x); for (auto& x : b.ap1) fn(*x); fn(*b.f0); fn(*b.f1); fn(*b.delay); }
  }
  void reset() override { each([](Node& n) { n.reset(); }); feedback = 0; }                        // :215-228 (the pre-delays are not reset)
  void set_sample_rate(double sr) override { each([sr](Node& n) { n.set_sample_rate(sr); }); }    // :230-242 (nor re-rated)
  static float mono(Node& n, float x) { float y; n.tick(&x, &y); return y; }
  void tick(const float* in, float* out) override {  // :244-274
    float v0 = feedback, o0 = 0, o1 = 0;
    float in0 = mono(*pre[0], in[0] * 0.5f); in0 = mono(*pre[1], in0);
    float in1 = mono(*pre[2], in[1] * 0.5f); in1 = mono(*pre[3], in1);
    for (auto& b : block) {
      v0 = mono(*b.delay, v0);
      v0 = mono(*b.ap0[0], a * v0 + in0); v0 = mono(*b.ap0[1], v0); v0 = mono(*b.ap0[2], v0); v0 = mono(*b.ap0[3], v0);
      v0 = mono(*b.f0, v0); o0 = v0;
      v0 = mono(*b.ap1[0], a * v0 + in1); v0 = mono(*b.ap1[1], v0); v0 = mono(*b.ap1[2], v0); v0 = mono(*b.ap1[3], v0);
      v0 = mono(*b.f1, v0); o1 = v0;
    }
    feedback = v0;
    out[0] = o0; out[1] = o1;
  }
  Node* clone() const override { return new Reverb85(*this); }
};
// ---- src/filter.rs (F = f32, the prelude32 instantiation): one-pole family
// kind 0 Lowpole (ID 18, :19-99), 1 Highpole (ID 47, :353-430), 2 Allpole (ID 46, :269-350), 3 DCBlock (ID 22, :102-175), 4 Pinkpass (ID 26, :178-262)
struct OnePole : Node {
  int kind, nin; float param, coeff = 0, sr = (float)DEFAULT_SR, x1 = 0, y1 = 0, b[7] = {0, 0, 0, 0, 0, 0, 0};
  OnePole(int kind_, float param_, int nin_) : kind(kind_), nin(nin_), param(param_) { set_param(param_); }
  void set_param(float p) {
    const float TAU = 6.28318548202514648f;
    param = p;
    if (kind == 0 || kind == 1) coeff = m::expf_(-TAU * p / sr);            // exp(-TAU * cutoff / sample_rate)
    else if (kind == 2) coeff = (1.0f - p) / (1.0f + p);                    // eta
    else if (kind == 3) coeff = 1.0f - TAU / sr * p;
  }
  int inputs() const override { return nin; } int outputs() const override { return 1; }
  uint64_t id() const override { static const uint64_t ids[5] = {18, 47, 46, 22, 26}; return ids[kind]; }
  void reset() override { x1 = y1 = 0; for (float& v : b) v = 0; }
  void set_sample_rate(double s) override { sr = (float)s; if (kind != 2 && kind != 4) set_param(param); }
  void tick(const float* in, float* out) override {
    if (nin > 1) { if (kind == 2) set_param(in[1]); else if (in[1] != param) set_param(in[1]); }
    const float x = in[0];
    if (kind == 0) { y1 = (1.0f - coeff) * x + coeff * y1; out[0] = y1; }
    else if (kind == 1) { float y0 = coeff * (y1 + x - x1); x1 = x; y1 = y0; out[0] = y0; }
    else if (kind == 2) { float y0 = coeff * (x - y1) + x1; x1 = x; y1 = y0; out[0] = y0; }
    else if (kind == 3) { float y0 = x - x1 + coeff * y1; x1 = x; y1 = y0; out[0] = y0; }
    else {
      b[0] = (float)0.99886 * b[0] + x * (float)0.0555179;
      b[1] = (float)0.99332 * b[1] + x * (float)0.0750759;
      b[2] = (float)0.96900 * b[2] + x * (float)0.1538520;
      b[3] = (float)0.86650 * b[3] + x * (float)0.3104856;
      b[4] = (float)0.55000 * b[4] + x * (float)0.5329522;
      b[5] = (float)-0.7616 * b[5] - x * (float)0.0168980;
      out[0] = (b[0] + b[1] + b[2] + b[3] + b[4] + b[5] + b[6] + x * (float)0.5362) * (float)0.115830421;
      b[6] = x * (float)0.115926;
    }
  }
  void set(const Setting& s) override {
    if ((kind == 0 || kind == 1 || kind == 3) && s.kind == P_CENTER) set_param(s.v[0]);
    else if (kind == 2 && s.kind == P_DELAY) set_param(s.v[0]);
  }
  FO_CLONE(OnePole)
};
// ---- src/oscillator.rs:318-438 Rossler (ID 73) and Lorenz (ID 74) chaotic oscillators (explicit Euler, input = frequency)
struct Chaos : Node {
  int kind; float x = 0, y = 1, z = 1, sr = (float)DEFAULT_SR; uint64_t hash = 0;
  explicit Chaos(int k) : kind(k) { reset(); }
  int inputs() const override { return 1; } int outputs() const override { return 1; }
  uint64_t id() const override { return kind == 0 ? 73 : 74; }
  void reset() override { const float t = (float)rnd1(hash); x = 0.0f * (1.0f - t) + 1.0f * t; y = 1.0f; z = 1.0f; }
  void set_sample_rate(double s) override { sr = (float)s; }
  void tick(const float* in, float* out) override {
    if (kind == 0) {
      const float dx = -y - z, dy = x + 0.15f * y, dz = 0.2f + z * (x - 10.0f), dt = 2.91f * in[0] / sr;
      x += dx * dt; y += dy * dt; z += dz * dt;
      out[0] = x * 0.05757f;
    } else {
      const float dx = 10.0f * (y - x), dy = x * (28.0f - z) - y, dz = x * y - (8.0f / 3.0f) * z, dt = in[0] / sr;
      x += dx * dt; y += dy * dt; z += dz * dt;
      out[0] = x * 0.05107f;
    }
  }
  void set_hash(uint64_t h) override { hash = h; reset(); }
  FO_CLONE(Chaos)
};
// ---- src/dynamics.rs:245-315 Declick<f32> (ID 23): smooth5 fade-in over the first `duration` seconds
inline float smooth5f(float x) { return ((x * 6.0f - 15.0f) * x + 10.0f) * x * x * x; }   // src/math.rs:418-420
struct Declick : Node {
  float t = 0, duration, sample_duration = 0;
  explicit Declick(float d) : duration(d) { set_sample_rate(DEFAULT_SR); }
  int inputs() const override { return 1; } int outputs() const override { return 1; }
  uint64_t id() const override { return 23; }
  void reset() override { t = 0; }
  void set_sample_rate(double sr) override { sample_duration = (float)(1.0 / sr); }
  void tick(const float* in, float* out) override {
    if (t < duration) { const float phase = (t - 0.0f) / (duration - 0.0f); const float value = smooth5f(phase); t += sample_duration; out[0] = in[0] * value; }
    else out[0] = in[0];
  }
  void process(int size, const float* in, float* out) override {  // :287-307: the phase is accumulated inside the block, t jumps by the block
    for (int i = 0; i < size; i++) out[i] = in[i];
    if (t < duration) {
      float phase = (t - 0.0f) / (duration - 0.0f);
      const float phase_d = sample_duration / duration;
      const float end_time = t + (float)size * sample_duration;
      const int end_index = duration < end_time ? (int)ceilf((duration - t) / sample_duration) : size;
      for (int i = 0; i < end_index && i < B; i++) { out[i] *= smooth5f(phase); phase += phase_d; }
      t = end_time;
    }
  }
  FO_CLONE(Declick)
};
// ---- src/follow.rs (F = f32): Follow (ID 24, :31-134) and AFollow (ID 29, :137-270): three one-pole smoothers in series
inline double halfway_coeff(double samples) {  // :17-23
  double r0 = log(fmax(1.0, samples)) - 0.861624594696583;
  double r1 = 1.0 / (1.0 + exp(0.0 - r0));
  double r2 = r1 * 1.13228543863477 - 0.1322853859;
  return 1.0 - fmin(0.9999999, r2);
}
struct Follower : Node {
  bool asym; float atime, rtime, acoeff = 0, rcoeff = 0, anow = 1, rnow = 1, v1 = 0, v2 = 0, v3 = 0, sr = 0;
  Follower(bool asym_, float a, float r) : asym(asym_), atime(a), rtime(r) { reset(); set_sample_rate(DEFAULT_SR); }
  void set_time(float a, float r) {
    atime = a; rtime = r;
    acoeff = (float)halfway_coeff((double)(atime * sr));
    rcoeff = (float)halfway_coeff((double)(rtime * sr));
    if (anow < 1.0f) { anow = acoeff; rnow = rcoeff; }
  }
  int inputs() const override { return 1; } int outputs() const override { return 1; }
  uint64_t id() const override { return asym ? 29 : 24; }
  void reset() override { v1 = v2 = v3 = 0; anow = rnow = 1.0f; }
  void set_value(float x) { v1 = v2 = v3 = x; }   // src/follow.rs:198-202
  void set_sample_rate(double s) override { sr = (float)s; set_time(atime, rtime); }
  static float pole2(float in, float cur, float a, float r) { return cur + fmaxf(0.0f, in - cur) * a - fmaxf(0.0f, cur - in) * r; }
  void tick(const float* in, float* out) override {
    if (asym) {
      v1 = pole2(in[0], v1, anow, rnow); v2 = pole2(v1, v2, anow, rnow); v3 = pole2(v2, v3, anow, rnow);
    } else {
      const float rc = 1.0f - anow;
      v1 = anow * in[0] + rc * v1; v2 = anow * v1 + rc * v2; v3 = anow * v2 + rc * v3;
    }
    anow = acoeff; rnow = rcoeff;
    out[0] = v3;
  }
  void set(const Setting& s) override {
    if (!asym && s.kind == P_TIME) set_time(s.v[0], s.v[0]);
    else if (asym && s.kind == P_ATTACK_RELEASE) set_time(s.v[0], s.v[1]);
  }
  FO_CLONE(Follower)
};
// ---- src/shape.rs Shaper<S> (ID 42): kind 0 Clip(h), 1 ClipTo(lo, hi), 2 Tanh(h), 3 Softsign(h), 4 Crush(levels), 5 SoftCrush(levels).
// `tick` uses Shape::shape, the block path Shape::simd on f32x8 groups — they differ for Softsign (|x|*h vs |x*h|), Crush
// (f32::round = half away from zero vs wide's round-to-even) and SoftCrush (libm floor vs F32x::floor, src/lib.rs:326-328).
struct Shaper : Node {
  int kind; float p0, p1;
  Shaper(int k, float a, float b) : kind(k), p0(a), p1(b) {}
  int inputs() const override { return 1; } int outputs() const override { return 1; }
  uint64_t id() const override { return 42; }
  float shape(float x) const {
    switch (kind) {
      case 0: return fminf(fmaxf(x * p0, -1.0f), 1.0f);
      case 1: return fminf(fmaxf(x, p0), p1);
      case 2: return m::tanhf_(x * p0);
      case 3: { float v = x * p0; return v / (1.0f + fabsf(v)); }
      case 4: return roundf(x * p0) / p0;
      default: { float v = x * p0, y = floorf(v); return (y + smooth9f(v - y)) / p0; }
    }
  }
  float simd(float x) const {
    switch (kind) {
      case 3: return x * p0 / (1.0f + fabsf(x) * p0);
      case 4: return wide_roundf(x * p0) / p0;
      case 5: { float v = x * p0, y = wide_floorf(v); return (y + smooth9f(v - y)) / p0; }
      default: return shape(x);
    }
  }
  void tick(const float* in, float* out) override { out[0] = shape(in[0]); }
  void process(int size, const float* in, float* out) override {  // :238-243
    const int full = size & ~7;
    for (int i = 0; i < full; i++) out[i] = simd(in[i]);
    process_remainder(size, in, out);
  }
  FO_CLONE(Shaper)
};
// ---- src/biquad.rs:494-920 nonlinear biquads (F = f32): FbBiquad (88) / FixedFbBiquad (90), DirtyBiquad (89) / FixedDirtyBiquad (91)
// mode 0 resonator, 1 lowpass, 2 highpass, 3 bell; the waveshaper is one of the Shaper kinds, always through Shape::shape.
struct NlBiquad : Node {
  bool fb; int mode, nin; Shaper shaper; BiquadCoefs c; float sr = (float)DEFAULT_SR, center = 440.0f, q = 1.0f, gain = 1.0f, s1 = 0, s2 = 0;
  NlBiquad(bool fb_, int mode_, int shape_kind, float p0, float p1, int nin_, float center_, float q_, float gain_)
      : fb(fb_), mode(mode_), nin(nin_), shaper(shape_kind, p0, p1) {
    update();                                   // new(): default parameters at the default rate
    if (nin == 1) { center = center_; q = q_; gain = gain_; update(); }   // dbell_hz etc.: set_center_q[_gain] after construction
  }
  void update() {
    switch (mode) { case 0: c = biquad_resonator(sr, center, q); break; case 1: c = biquad_lowpass(sr, center, q); break;
      case 2: c = biquad_highpass(sr, center, q); break; default: c = biquad_bell(sr, center, q, gain); }
  }
  int inputs() const override { return nin; } int outputs() const override { return 1; }
  uint64_t id() const override { return fb ? (nin == 1 ? 90 : 88) : (nin == 1 ? 91 : 89); }
  void reset() override { s1 = s2 = 0; }
  void set_sample_rate(double s) override { sr = (float)s; update(); }
  void tick(const float* in, float* out) override {
    if (nin == 3) {
      const float dc = in[1] - center, dq = in[2] - q;
      if (dc * dc + dq * dq != 0.0f) { center = in[1]; q = in[2]; update(); }
    } else if (nin == 4) {
      const float dc = in[1] - center, dq = in[2] - q, dg = in[3] - gain;
      if (dc * dc + dq * dq + dg * dg != 0.0f) { center = in[1]; q = in[2]; gain = in[3]; update(); }
    }
    const float x0 = in[0], y0 = c.b0 * x0 + s1;
    if (fb) { const float f = shaper.shape(y0); s1 = s2 + c.b1 * x0 - f * c.a1; s2 = c.b2 * x0 - f * c.a2; }
    else { s1 = shaper.shape(s2 + c.b1 * x0 - y0 * c.a1); s2 = shaper.shape(c.b2 * x0 - y0 * c.a2); }
    out[0] = y0;
  }
  void set(const Setting& s) override {
    if (nin != 1) return;
    if (s.kind == P_CENTER) { center = s.v[0]; update(); }
    else if (s.kind == P_CENTER_Q) { center = s.v[0]; q = s.v[1]; update(); }
    else if (s.kind == P_CENTER_Q_GAIN) { center = s.v[0]; q = s.v[1]; gain = s.v[2]; update(); }
  }
  FO_CLONE(NlBiquad)
};
// ---- src/convolve.rs:9-59 Convolver (ID 100): y = x * h. The reference delegates to the un-vendored crate fft-convolver 0.3.0
// (uniformly partitioned FFT overlap-add, block 64); what is restated here is the quantity that algorithm computes — the
// linear convolution — accumulated in f64 and rounded once, which the FFT form matches to ~1e-6 of the signal scale.
// Pin: tests/test_basic.rs:698-711 (impulse through [1, .75, .5, .25], tolerance 1e-4).
struct Convolver : Node {
  std::vector<float> h, hist; size_t i = 0;
  explicit Convolver(std::vector<float> response) : h(std::move(response)) { if (h.empty()) h.push_back(0.0f); hist.assign(h.size(), 0.0f); }
  int inputs() const override { return 1; } int outputs() const override { return 1; }
  uint64_t id() const override { return 100; }
  void reset() override { std::fill(hist.begin(), hist.end(), 0.0f); i = 0; }
  void tick(const float* in, float* out) override {
    const size_t K = h.size();
    hist[i] = in[0];
    double acc = 0.0;
    for (size_t k = 0; k < K; k++) acc += (double)h[k] * (double)hist[(i + K - k) % K];
    i = (i + 1) % K;
    out[0] = (float)acc;
  }
  FO_CLONE(Convolver)
};
// ---- src/shared.rs:84-131 Var (ID 68): outputs a shared control value, sampled once per block; here the value is a Setting
struct Var : Node {
  float value;
  explicit Var(float v) : value(v) {}
  int inputs() const override { return 0; } int outputs() const override { return 1; }
  uint64_t id() const override { return 68; }
  void tick(const float*, float* out) override { out[0] = value; }
  void set(const Setting& s) override { if (s.kind == P_VALUE) value = s.v[0]; }
  FO_CLONE(Var)
};

// ---- src/denormal.rs:5-21 prevent_denormals: _mm_setcsr(0x9fc0) = FTZ + DAZ, process-wide and sticky.
inline bool& denormal_emulation_enabled() { static bool e = true; return e; }
inline void prevent_denormals() { if (denormal_emulation_enabled()) _mm_setcsr(0x9fc0); }

// ---- src/feedback.rs:17-66 FrameHadamard, :68-178 Feedback<N,X,U> (ID 11)
inline void hadamard(float* v, int n) {
  for (int h = 1; h < n; h *= 2)
    for (int i = 0; i < n; i += h * 2)
      for (int j = i; j < i + h; j++) { float x = v[j], y = v[j + h]; v[j] = x + y; v[j + h] = x - y; }
  const float z = (float)(1.0 / sqrt((double)n));
  for (int i = 0; i < n; i++) v[i] = v[i] * z;
}
struct Feedback : Node {
  Child x; bool had; std::vector<float> value;
  Feedback(Node* x_, bool hadamard_) : x(x_), had(hadamard_) {
    assert(x->inputs() == x->outputs());
    prevent_denormals();
    value.assign(x->inputs(), 0.0f);
    ctor_ping();
  }
  int inputs() const override { return x->inputs(); } int outputs() const override { return x->outputs(); }
  uint64_t id() const override { return 11; }
  void reset() override { x->reset(); std::fill(value.begin(), value.end(), 0.0f); }
  void set_sample_rate(double sr) override { x->set_sample_rate(sr); }
  void tick(const float* in, float* out) override {
    const int n = inputs(); float t[256];
    for (int c = 0; c < n; c++) t[c] = in[c] + value[c];
    x->tick(t, out);
    for (int c = 0; c < n; c++) value[c] = out[c];
    if (had) hadamard(value.data(), n);
  }
  void process(int size, const float* in, float* out) override {  // :136-146: ticks the inner graph
    const int n = inputs(); float t[256], o[256];
    for (int i = 0; i < size; i++) {
      for (int c = 0; c < n; c++) t[c] = in[c * B + i] + value[c];
      x->tick(t, o);
      for (int c = 0; c < n; c++) value[c] = o[c];
      if (had) hadamard(value.data(), n);
      for (int c = 0; c < n; c++) out[c * B + i] = o[c];
    }
  }
  AttoHash ping(bool probe, AttoHash h) override { return x->ping(probe, h.hash(id())); }
  FO_CLONE(Feedback)
};

// ---- src/feedback.rs:316-481 FeedbackUnit (ID 79): feedback loop with an integrated delay of round(delay*sr) >= 1 samples.
// Blocks no longer than the delay run the inner unit's BLOCK path on (input + delayed output); longer ones go sample by sample.
struct FeedbackUnit : Node {
  Child x; int channels; double sample_rate = 0.0, delay; size_t samples = 0, mask = 0, index = 0;
  std::vector<std::vector<float>> feedback;
  FeedbackUnit(double delay_, Node* x_) : x(x_), channels(x_->inputs()), delay(delay_) {
    assert(x->inputs() == x->outputs());
    prevent_denormals();
    feedback.assign(channels, std::vector<float>());
    set_sample_rate(DEFAULT_SR);
  }
  int inputs() const override { return channels; } int outputs() const override { return channels; }
  uint64_t id() const override { return 79; }
  size_t read_index(size_t d) const { return (index + mask + 1 - d) & mask; }
  void reset() override { for (auto& f : feedback) std::fill(f.begin(), f.end(), 0.0f); x->reset(); index = 0; }
  void set_sample_rate(double sr) override {
    if (sample_rate != sr) {
      sample_rate = sr;
      x->set_sample_rate(sr);
      samples = (size_t)fmax(round(delay * sr), 1.0);
      size_t p2 = 1; while (p2 < samples) p2 <<= 1;
      mask = p2 - 1;
      for (auto& f : feedback) { std::fill(f.begin(), f.end(), 0.0f); f.resize(p2, 0.0f); }
      index = 0;
    }
  }
  void tick(const float* in, float* out) override {
    float t[256];
    const size_t ri = read_index(samples);
    for (int c = 0; c < channels; c++) t[c] = in[c] + feedback[c][ri];
    x->tick(t, out);
    for (int c = 0; c < channels; c++) feedback[c][index] = out[c];
    index = (index + 1) & mask;
  }
  void process(int size, const float* in, float* out) override {
    if ((size_t)size <= samples) {
      std::vector<float> buf((size_t)channels * B, 0.0f);
      for (int c = 0; c < channels; c++) {
        size_t ri = read_index(samples);
        for (int i = 0; i < size; i++) { buf[c * B + i] = in[c * B + i] + feedback[c][ri]; ri = (ri + 1) & mask; }
      }
      x->process(size, buf.data(), out);
      for (int c = 0; c < channels; c++) {
        size_t wi = index;
        for (int i = 0; i < size; i++) { feedback[c][wi] = out[c * B + i]; wi = (wi + 1) & mask; }
      }
    } else {
      float t[256], o[256];
      size_t ri = read_index(samples), wi = index;
      for (int i = 0; i < size; i++) {
        for (int c = 0; c < channels; c++) t[c] = in[c * B + i] + feedback[c][ri];
        x->tick(t, o);
        for (int c = 0; c < channels; c++) { out[c * B + i] = o[c]; feedback[c][wi] = o[c]; }
        ri = (ri + 1) & mask; wi = (wi + 1) & mask;
      }
    }
    index = (index + (size_t)size) & mask;
  }
  AttoHash ping(bool probe, AttoHash h) override { return x->ping(probe, h.hash(id())); }
  FO_CLONE(FeedbackUnit)
};

// ---- src/oscillator.rs:440-760 Ramp (ID 94), PolySaw (95), PolySquare (96), PolyPulse (97): phase oscillators, tick only
inline float polyblep(float t, float dt) {  // :510-521
  if (t < dt) { float z = t / dt; return z + z - z * z - 1.0f; }
  else if (t > 1.0f - dt) { float z = (t - 1.0f) / dt; return z + z + z * z + 1.0f; }
  return 0.0f;
}
struct PhaseOsc : Node {
  int kind;  // 0 ramp, 1 poly_saw, 2 poly_square, 3 poly_pulse
  float phase = 0, sample_duration = 0; uint64_t hash = 0; bool has_phase = false; float initial_phase = 0;
  explicit PhaseOsc(int k) : kind(k) { reset(); set_sample_rate(DEFAULT_SR); }
  int inputs() const override { return kind == 3 ? 2 : 1; } int outputs() const override { return 1; }
  uint64_t id() const override { return 94 + (uint64_t)kind; }
  void reset() override { phase = has_phase ? initial_phase : (float)rnd1(hash); }
  void set_sample_rate(double sr) override { sample_duration = (float)(1.0 / sr); }
  void tick(const float* in, float* out) override {
    float p = phase;
    float delta = in[0] * sample_duration;
    phase += delta;
    phase -= floorf(phase);
    if (kind == 0) { out[0] = p; return; }
    if (kind == 1) { out[0] = 2.0f * p - 1.0f - polyblep(p, delta); return; }
    float width = kind == 2 ? 0.5f : in[1];
    float square = p < width ? 1.0f : -1.0f;
    float half = p - width;
    out[0] = square + polyblep(p, delta) - polyblep(half - floorf(half), delta);
  }
  void set(const Setting& s) override { if (s.kind == P_PHASE) { has_phase = true; initial_phase = s.v[0]; } }
  void set_hash(uint64_t h) override { hash = h; reset(); }
  FO_CLONE(PhaseOsc)
};

// ---- src/oscillator.rs:104-208 Dsf<N> (ID 55): discrete summation formula oscillator (Moorer 1976), N = 1 or 2 inputs
inline float dsf_formula(float f, float d, float r, float n) {  // :105-112, f32 instantiation: libm sinf / cosf / powf
  return (m::sinf_(f) - r * m::sinf_(f - d) - m::powf_(r, n + 1.0f) * (m::sinf_(f + (n + 1.0f) * d) - r * m::sinf_(f + n * d))) / (1.0f + r * r - 2.0f * r * m::cosf_(d));
}
struct Dsf : Node {
  int nin; float phase = 0, roughness, harmonic_spacing, sample_duration = 0; uint64_t hash = 0; bool has_phase = false; float initial_phase = 0;
  Dsf(int nin_, float spacing, float rough) : nin(nin_), roughness(rough), harmonic_spacing(spacing) { reset(); set_sample_rate(DEFAULT_SR); set_roughness(rough); }
  void set_roughness(float r) { roughness = fminf(fmaxf(r, 0.0001f), 0.9999f); }  // clamp(0.0001, 0.9999, r) = r.max(lo).min(hi)
  int inputs() const override { return nin; } int outputs() const override { return 1; }
  uint64_t id() const override { return 55; }
  void reset() override { phase = has_phase ? initial_phase : (float)rnd1(hash); }
  void set_sample_rate(double sr) override { sample_duration = (float)(1.0 / sr); }
  void tick(const float* in, float* out) override {  // :171-187
    if (nin > 1) set_roughness(in[1]);
    phase += in[0] * sample_duration;
    phase -= floorf(phase);
    const float n = floorf(22050.0f / in[0] / harmonic_spacing);
    const float TAU_F = 6.28318548202514648f;   // f32::TAU
    out[0] = dsf_formula(phase * TAU_F, phase * TAU_F * harmonic_spacing, roughness, n);
  }
  void set(const Setting& s) override {
    if (s.kind == P_ROUGHNESS) set_roughness(s.v[0]);
    else if (s.kind == P_PHASE) { has_phase = true; initial_phase = s.v[0]; }
  }
  void set_hash(uint64_t h) override { hash = h; reset(); }
  FO_CLONE(Dsf)
};

// ---- src/noise.rs:11-148 Mls (ID 19): maximum length sequence
static const uint32_t MLS_POLY[31] = {
    0b1, 0b11, 0b110, 0b1100, 0b10100, 0b110000, 0b1001000, 0b10111000, 0b100010000, 0b1001000000, 0b10100000000, 0b110010100000,
    0b1101100000000, 0b11000010001000, 0b110000000000000, 0b1101000000001000, 0b10010000000000000, 0b100000010000000000,
    0b1100011000000000000, 0b10010000000000000000, 0b101000000000000000000, 0b1100000000000000000000, 0b10000100000000000000000,
    0b111000010000000000000000, 0b1001000000000000000000000, 0b10000000000000000000100011, 0b100000000000000000000010011,
    0b1001000000000000000000000000, 0b10100000000000000000000000000, 0b100000000000000000000000101001, 0b1001000000000000000000000000000};
struct Mls : Node {
  uint32_t n, s; bool has_seed = false; uint64_t seed = 0, hash = 0;
  explicit Mls(uint32_t n_) : n(n_), s((1u << n_) - 1u) {}
  int inputs() const override { return 0; } int outputs() const override { return 1; }
  uint64_t id() const override { return 19; }
  void reset() override { uint64_t h = has_seed ? seed : hash; uint32_t sd = (uint32_t)(h ^ (h >> 32)); s = 1u + sd % ((1u << n) - 1u); }
  void tick(const float*, float* out) override {
    float value = (float)((s >> (n - 1)) & 1u);
    uint32_t fb = MLS_POLY[n - 1] & s;
    uint32_t parity = (uint32_t)__builtin_popcount(fb) & 1u;
    s = ((s << 1) | parity) & ((1u << n) - 1u);
    out[0] = value * 2.0f - 1.0f;
  }
  void set(const Setting& st) override { if (st.kind == P_SEED) { has_seed = true; seed = st.seed; } }
  void set_hash(uint64_t h) override { hash = h; reset(); }
  FO_CLONE(Mls)
};

// ---- src/audionode.rs:2839-2873 Impulse<N> (ID 81)
struct Impulse : Node {
  int n; float value = 1.0f;
  explicit Impulse(int n_) : n(n_) {}
  int inputs() const override { return 0; } int outputs() const override { return n; }
  uint64_t id() const override { return 81; }
  void reset() override { value = 1.0f; }
  void tick(const float*, float* out) override { for (int c = 0; c < n; c++) out[c] = value; value = 0.0f; }
  FO_CLONE(Impulse)
};

// ---- src/math.rs:327-333 spline (Catmull-Rom), T = f32
inline float splinef(float y0, float y1, float y2, float y3, float x) {
  return y1 + x * 0.5f * (y2 - y0 + x * (2.0f * y0 - 5.0f * y1 + 4.0f * y2 - y3 + x * (3.0f * (y1 - y2) + y3 - y0)));
}
// ---- src/delay.rs:141-286 Tap<N> (ID 50) and :379-505 TapLinear<N> (ID 54). The block path (:238-279) writes the 8 inputs of a
// SIMD group first and reads relative to each lane's own write position; since every tap is >= 1.00001 samples that equals the tick path.
struct Tap : Node {
  int ntaps; bool linear; std::vector<float> buffer; size_t i = 0; float sr = 0, min_delay, max_delay, min_c = 0, max_c = 0;
  Tap(int ntaps_, bool linear_, float mn, float mx) : ntaps(ntaps_), linear(linear_), min_delay(mn), max_delay(mx) { assert(mn >= 0.0f && mn <= mx); set_sample_rate(DEFAULT_SR); }
  int inputs() const override { return ntaps + 1; } int outputs() const override { return 1; }
  uint64_t id() const override { return linear ? 54 : 50; }
  void reset() override { i = 0; std::fill(buffer.begin(), buffer.end(), 0.0f); }
  void set_sample_rate(double s) override {
    float f = (float)s;
    if (sr != f) {
      sr = f;
      min_c = fmaxf(min_delay, 1.00001f / f); max_c = fmaxf(max_delay, 1.00001f / f);
      float bl = linear ? ceilf(max_delay * f) + 2.0f : ceilf(max_delay * f) + 3.0f + 8.0f;
      size_t n = (size_t)bl, p2 = 1; while (p2 < n) p2 <<= 1;
      buffer.assign(p2, 0.0f);
      reset();
    }
  }
  void tick(const float* in, float* out) override {
    const size_t mask = buffer.size() - 1;
    buffer[i] = in[0];
    float o = 0.0f;
    for (int t = 1; t <= ntaps; t++) {
      float tap = (linear ? fminf(fmaxf(in[t], min_delay), max_delay) : fminf(fmaxf(in[t], min_c), max_c)) * sr;
      size_t tf = (size_t)tap;
      size_t i1 = (i - tf) & mask;
      float d = tap - (float)tf;
      if (linear) { size_t i2 = (i1 - 1) & mask; o += lerpf(buffer[i1], buffer[i2], d); }
      else { size_t i0 = (i1 + 1) & mask, i2 = (i1 - 1) & mask, i3 = (i1 - 2) & mask; o += splinef(buffer[i0], buffer[i1], buffer[i2], buffer[i3], d); }
    }
    i = (i + 1) & mask;
    out[0] = o;
  }
  FO_CLONE(Tap)
};

// ---- src/feedback.rs:180-314 Feedback2<N,X,Y,U> (ID 66): out = x(in + value); value = U(y(out))
struct Feedback2 : Node {
  Child x, y; bool had; std::vector<float> value;
  Feedback2(Node* x_, Node* y_, bool hadamard_) : x(x_), y(y_), had(hadamard_) {
    assert(x->inputs() == x->outputs() && y->inputs() == y->outputs() && x->inputs() == y->inputs());
    prevent_denormals();
    value.assign(x->inputs(), 0.0f);
    ctor_ping();
  }
  int inputs() const override { return x->inputs(); } int outputs() const override { return x->outputs(); }
  uint64_t id() const override { return 66; }
  void reset() override { x->reset(); y->reset(); std::fill(value.begin(), value.end(), 0.0f); }
  void set_sample_rate(double sr) override { x->set_sample_rate(sr); y->set_sample_rate(sr); }
  void tick(const float* in, float* out) override {
    const int n = inputs(); float t[256], u[256];
    for (int c = 0; c < n; c++) t[c] = in[c] + value[c];
    x->tick(t, out);
    y->tick(out, u);
    for (int c = 0; c < n; c++) value[c] = u[c];
    if (had) hadamard(value.data(), n);
  }
  AttoHash ping(bool probe, AttoHash h) override { return y->ping(probe, x->ping(probe, h.hash(id()))); }
  FO_CLONE(Feedback2)
};

// ---- src/pan.rs:12-91 Panner<N> (ID 49)
inline void pan_weights(float value, float& l, float& r) {
  float angle = (clamp11f(value) + 1.0f) * (3.14159274101257324f * 0.25f);
  l = m::cosf_(angle); r = m::sinf_(angle);
}
struct Panner : Node {
  int nin; float lw, rw;
  Panner(float value, int nin_) : nin(nin_) { pan_weights(value, lw, rw); }
  int inputs() const override { return nin; } int outputs() const override { return 2; }
  uint64_t id() const override { return 49; }
  void tick(const float* in, float* out) override {
    if (nin > 1) pan_weights(in[1], lw, rw);
    out[0] = lw * in[0]; out[1] = rw * in[0];
  }
  void process(int size, const float* in, float* out) override {
    if (nin == 1) {
      for (int i = 0; i < simd_items(size) * 8; i++) { out[i] = in[i] * lw; out[B + i] = in[i] * rw; }
    } else {
      for (int i = 0; i < size; i++) { pan_weights(in[B + i], lw, rw); out[i] = in[i] * lw; out[B + i] = in[i] * rw; }
    }
  }
  void set(const Setting& s) override { if (s.kind == P_PAN) pan_weights(s.v[0], lw, rw); }
  FO_CLONE(Panner)
};

// ---- src/pan.rs:95-160 Mixer<M, N> (ID 84): constant matrix, tick only
struct Mixer : Node {
  int m, n; std::vector<float> w;
  Mixer(int m_, int n_, const float* w_) : m(m_), n(n_), w(w_, w_ + (size_t)m_ * n_) {}
  int inputs() const override { return m; } int outputs() const override { return n; }
  uint64_t id() const override { return 84; }
  void tick(const float* in, float* out) override {
    for (int i = 0; i < n; i++) { float v = 0.0f; for (int j = 0; j < m; j++) v += in[j] * w[(size_t)i * m + j]; out[i] = v; }
  }
  FO_CLONE(Mixer)
};

// ---- src/dynamics.rs:56-243 ReduceBuffer<f32, Maximum> + Limiter<N> (ID 25); the follower is AFollow<f32> (src/follow.rs:137-245)
struct Limiter : Node {
  int n; double lookahead, sample_rate; Follower follower;
  std::vector<float> tree; size_t length = 0, leaf_offset = 0; std::vector<float> buffer; size_t filled = 0, index = 0;
  void new_buffer() {
    double r = round(sample_rate * lookahead);
    length = r < 1.0 ? 1 : (size_t)r;
    leaf_offset = 1; while (leaf_offset < length) leaf_offset <<= 1;
    tree.assign(leaf_offset + length + (length & 1), 0.0f);
  }
  Limiter(int n_, float attack, float release) : n(n_), lookahead((double)attack), sample_rate(DEFAULT_SR), follower(true, attack * 0.4f, release * 0.4f) {
    follower.set_sample_rate(sample_rate); new_buffer(); buffer.assign((size_t)n * length, 0.0f);
  }
  int inputs() const override { return n; } int outputs() const override { return n; }
  uint64_t id() const override { return 25; }
  void reset() override { set_sample_rate(sample_rate); }
  void set_sample_rate(double sr) override {   // :185-195 (the follower is NOT reset: only its coefficients are recomputed)
    index = 0; sample_rate = sr; new_buffer(); follower.set_sample_rate(sr);
    buffer.assign((size_t)n * length, 0.0f); filled = 0;
  }
  void reduce_set(size_t idx, float value) {   // :106-114
    size_t i = leaf_offset + idx;
    tree[i] = value;
    while (i > 1) { float reduced = fmaxf(tree[i], tree[i ^ 1]); i >>= 1; tree[i] = reduced; }
  }
  void tick(const float* in, float* out) override {   // :197-222
    float amplitude = 0.0f;
    for (int k = 0; k < n; k++) amplitude = fmaxf(amplitude, fabsf(in[k]));
    reduce_set(index, amplitude);
    if (filled < length) {
      for (int k = 0; k < n; k++) { buffer[(size_t)k * length + filled] = in[k]; out[k] = 0.0f; }
      filled++;
      if (filled == length) follower.set_value(tree[1]);
    } else {
      float x = fmaxf(1.0f, tree[1] * 1.10f), y;
      follower.tick(&x, &y);
      const float limit = follower.v3, g = 1.0f / limit;
      for (int k = 0; k < n; k++) { float* slot = &buffer[(size_t)k * length + index]; out[k] = *slot * g; *slot = in[k]; }
    }
    index += 1; if (index >= length) index = 0;
  }
  FO_CLONE(Limiter)
};
// ---- src/envelope.rs:14-183 Envelope<F, E, R> (ID 14): the closure is a live callback here, exactly as in the reference
typedef void (*EnvelopeFn)(double t, double* out, void* user);
template <class F> struct Envelope : Node {
  EnvelopeFn fn; void* user; int nout;
  F t = 0, t_0 = 0, t_1 = 0, interval, sample_duration = 0; uint64_t t_hash = 0, hash = 0;
  std::vector<float> value_0, value_1, value, value_d;
  Envelope(F iv, int n, EnvelopeFn f, void* u) : fn(f), user(u), nout(n), interval(iv), value_0(n, 0.0f), value_1(n, 0.0f), value(n, 0.0f), value_d(n, 0.0f) {
    set_sample_rate(DEFAULT_SR); reset();
  }
  void call(F at, std::vector<float>& into) { double o[16]; fn((double)at, o, user); for (int c = 0; c < nout; c++) into[c] = (float)o[c]; }
  void next_segment() {   // :63-82
    t_0 = t_1; value_0 = value_1;
    const F w = (F)rnd1(t_hash);
    const F next_interval = ((F)0.75f * ((F)1 - w) + (F)1.25f * w) * interval;
    t_1 = t_0 + next_interval;
    call(t_1, value_1);
    t_hash = t_hash * 6364136223846793005ull + 1ull;
    const F u = (t - t_0) / (t_1 - t_0);
    const F samples = next_interval / sample_duration;
    for (int c = 0; c < nout; c++) { value[c] = value_0[c] * (1.0f - (float)u) + value_1[c] * (float)u; value_d[c] = (value_1[c] - value_0[c]) / (float)samples; }
  }
  int inputs() const override { return 0; } int outputs() const override { return nout; }
  uint64_t id() const override { return 14; }
  void reset() override { t = 0; t_0 = 0; t_1 = 0; t_hash = hash; call(t_0, value_0); value_1 = value_0; }
  void set_sample_rate(double sr) override { sample_duration = (F)(1.0 / sr); }
  void tick(const float*, float* out) override {   // :117-126
    if (t >= t_1) next_segment();
    for (int c = 0; c < nout; c++) { out[c] = value[c]; value[c] += value_d[c]; }
    t += sample_duration;
  }
  void process(int size_, const float*, float* out) override {   // :128-157
    const size_t size = (size_t)size_;
    if (t >= t_1) next_segment();
    size_t i = 0;
    while (i < size) {
      const size_t left = (size_t)(long long)(sizeof(F) == 8 ? (double)ceil((double)((t_1 - t) / sample_duration)) : (double)ceilf((float)((t_1 - t) / sample_duration)));
      const size_t loop = std::min(size - i, left);
      for (int c = 0; c < nout; c++) { float v = value[c], d = value_d[c]; for (size_t o = 0; o < loop; o++) { out[c * B + i + o] = v; v += d; } value[c] = v; }
      i += loop;
      t += (F)(long long)loop * sample_duration;
      if (loop == left) next_segment();
    }
  }
  void set(const Setting& s) override { if (s.kind == P_INTERVAL) interval = (F)s.v[0]; }
  void set_hash(uint64_t h) override { hash = h; t_hash = h; }
  Node* clone() const override { return new Envelope<F>(*this); }
};

// ---- src/oversample.rs Oversampler<X> (ID 51): 2x oversampling around X with a 43-tap minimum-phase halfband (coefficients :344-388),
// restated as written: the window ends at the newest sample and meets the taps in table order; decimation loops over the INPUT channel
// count (:207); with an odd block size the last output sample is not written (0 here) and X processes one zero-input sample more per
// half. `wide` without AVX/FMA (the default x86-64 build): mul_add = mul then add; reduce_add = ((l0+l2)+(l1+l3)) per f32x4, low half
// + high half — the lane-sum association is restated from the crate's SSE path from memory (ulp-level parity unpinned, like libm).
static const float kHalfbandMin[43] = {
    4.73552339e-02f, 1.81988040e-01f, 3.49148434e-01f, 3.92748135e-01f, 2.18230867e-01f, -5.31842843e-02f, -1.79186566e-01f, -7.34488007e-02f,
    8.94524103e-02f, 1.00868556e-01f, -2.08681451e-02f, -8.82510989e-02f, -2.07640777e-02f, 6.22587555e-02f, 4.07776255e-02f, -3.52258090e-02f,
    -4.57407870e-02f, 1.27033444e-02f, 4.14376136e-02f, 3.30799834e-03f, -3.24608206e-02f, -1.27856355e-02f, 2.21659033e-02f, 1.67803711e-02f,
    -1.27406974e-02f, -1.68177367e-02f, 5.35518220e-03f, 1.44761581e-02f, -3.70651781e-04f, -1.11140183e-02f, -2.40622311e-03f, 7.71596027e-03f,
    3.48227062e-03f, -4.86763558e-03f, -3.45536353e-03f, 2.79880054e-03f, 2.86736431e-03f, -1.48746153e-03f, -2.11827989e-03f, 7.72684113e-04f,
    1.44384114e-03f, -4.49807048e-04f, -9.41945265e-04f};
inline float os_dec_coeff(int k) { return k < 5 ? 0.0f : kHalfbandMin[k - 5]; }                       // DECIMATING_COEFFS flattened, k = 0..47 (:395-457)
inline float os_even_coeff(int k) { return k < 2 ? 0.0f : kHalfbandMin[2 * (k - 2)]; }               // INTERPOLATING_EVEN_COEFFS, k = 0..23 (:460-492)
inline float os_odd_coeff(int k) { return k < 3 ? 0.0f : kHalfbandMin[2 * (k - 3) + 1]; }            // INTERPOLATING_ODD_COEFFS (:495-527)
inline float os_reduce8(const float* a) { return ((a[0] + a[2]) + (a[1] + a[3])) + ((a[4] + a[6]) + (a[5] + a[7])); }
inline void os_interpolate(const float* ring, size_t newest, float& even, float& odd) {                // :12-44
  const size_t start = newest + (129 - 3 * 8);
  float ae[8] = {0, 0, 0, 0, 0, 0, 0, 0}, ao[8] = {0, 0, 0, 0, 0, 0, 0, 0};
  for (int i = 0; i < 3; i++) for (int j = 0; j < 8; j++) {
    const float sm = ring[(start + (size_t)i * 8 + j) & 0x7f];
    ae[j] = sm * os_even_coeff(i * 8 + j) + ae[j];
    ao[j] = sm * os_odd_coeff(i * 8 + j) + ao[j];
  }
  even = os_reduce8(ae) * 2.0f; odd = os_reduce8(ao) * 2.0f;
}
inline float os_decimate(const float* ring, size_t last) {                                             // :46-66
  const size_t start = last + (129 - (43 / 8 + 1) * 8);
  float acc[8] = {0, 0, 0, 0, 0, 0, 0, 0};
  for (int i = 0; i < 6; i++) for (int j = 0; j < 8; j++) acc[j] = ring[(start + (size_t)i * 8 + j) & 0x7f] * os_dec_coeff(i * 8 + j) + acc[j];
  return os_reduce8(acc);
}
struct Oversampler : Node {
  Child x; int nin, nout; std::vector<float> inv, outv, inner_in, inner_out; size_t input_rb_index = 0, output_rb_index = 0;
  explicit Oversampler(Node* x_) : x(x_), nin(x_->inputs()), nout(x_->outputs()) {
    x->set_sample_rate(DEFAULT_SR * 2.0);
    AttoHash h = x->ping(true, AttoHash(51)); x->ping(false, h);
    inv.assign((size_t)std::max(1, nin) * 128, 0.0f); outv.assign((size_t)std::max(1, nout) * 128, 0.0f);
    inner_in.assign((size_t)std::max(1, nin) * B, 0.0f); inner_out.assign((size_t)std::max(1, nout) * B, 0.0f);
  }
  int inputs() const override { return nin; } int outputs() const override { return nout; }
  uint64_t id() const override { return 51; }
  void reset() override { x->reset(); std::fill(inv.begin(), inv.end(), 0.0f); std::fill(outv.begin(), outv.end(), 0.0f); }   // the ring positions keep running (:137-141)
  void set_sample_rate(double sr) override { x->set_sample_rate(sr * 2.0); }
  void tick(const float* in, float* out) override {   // :149-180
    float a[64], b[64], y[64];
    for (int c = 0; c < nin; c++) { inv[(size_t)c * 128 + input_rb_index] = in[c]; os_interpolate(&inv[(size_t)c * 128], input_rb_index, a[c], b[c]); }
    input_rb_index = (input_rb_index + 1) & 0x7f;
    x->tick(a, y);
    for (int c = 0; c < nout; c++) outv[(size_t)c * 128 + output_rb_index] = y[c];
    output_rb_index = (output_rb_index + 1) & 0x7f;
    x->tick(b, y);
    for (int c = 0; c < nout; c++) outv[(size_t)c * 128 + output_rb_index] = y[c];
    for (int c = 0; c < nout; c++) out[c] = os_decimate(&outv[(size_t)c * 128], output_rb_index);
    output_rb_index = (output_rb_index + 1) & 0x7f;
  }
  void process(int size, const float* in, float* out) override {   // :182-215
    std::fill(inner_in.begin(), inner_in.end(), 0.0f); std::fill(inner_out.begin(), inner_out.end(), 0.0f);   // BufferArray::new() per call
    if (size & 1) for (int c = 0; c < nout; c++) out[c * B + size - 1] = 0.0f;   // never written by the reference (see header)
    for (int c = nin; c < nout; c++) for (int i = 0; i < size; i++) out[c * B + i] = 0.0f;   // channels beyond the input count: never written either
    const int half = size / 2;
    for (int offset : {0, half}) {
      for (int i = 0; i < half; i++) {
        for (int c = 0; c < nin; c++) {
          inv[(size_t)c * 128 + input_rb_index] = in[c * B + i + offset];
          os_interpolate(&inv[(size_t)c * 128], input_rb_index, inner_in[c * B + 2 * i], inner_in[c * B + 2 * i + 1]);
        }
        input_rb_index = (input_rb_index + 1) & 0x7f;
      }
      x->process(size, inner_in.data(), inner_out.data());
      for (int i = 0; i < half; i++) {
        for (int c = 0; c < nin && c < nout; c++) {   // `for channel in 0..Self::Inputs::USIZE` as written
          outv[(size_t)c * 128 + output_rb_index] = inner_out[c * B + 2 * i];
          const size_t next = (output_rb_index + 1) & 0x7f;
          outv[(size_t)c * 128 + next] = inner_out[c * B + 2 * i + 1];
          out[c * B + i + offset] = os_decimate(&outv[(size_t)c * 128], next);
        }
        output_rb_index = (output_rb_index + 2) & 0x7f;
      }
    }
  }
  void set(const Setting& s) override { (void)s; }
  AttoHash ping(bool probe, AttoHash h) override { return x->ping(probe, h.hash(id())); }
  FO_CLONE(Oversampler)
};

// ---- src/dynamics.rs:316-437 Meter / MeterState / MeterNode (ID 61); kind 0 Sample, 1 Peak(timescale), 2 Rms(timescale)
struct MeterNode : Node {
  int kind; double timescale; float smoothing = 0, state = 0;
  MeterNode(int k, double t) : kind(k), timescale(t) { set_sample_rate(DEFAULT_SR); }
  int inputs() const override { return 1; } int outputs() const override { return 1; }
  uint64_t id() const override { return 61; }
  void reset() override { state = 0; }
  void set_sample_rate(double sr) override { if (kind != 0) smoothing = (float)pow(0.5, 1.0 / (timescale * sr)); }
  void tick(const float* in, float* out) override {
    const float v = in[0];
    if (kind == 0) { state = v; out[0] = state; }
    else if (kind == 1) { state = fmaxf(state * smoothing, fabsf(v)); out[0] = state; }
    else { state = state * smoothing + (v * v) * (1.0f - smoothing); out[0] = sqrtf(state); }
  }
  FO_CLONE(MeterNode)
};
// ---- src/wave.rs:739-797 WavePlayer (ID 65): plays one channel of a wave from start to end, optionally jumping to a loop point
struct WavePlayer : Node {
  std::shared_ptr<const std::vector<float>> wave; size_t index, start_point, end_point; bool has_loop; size_t loop_point;
  WavePlayer(std::shared_ptr<const std::vector<float>> w, size_t s, size_t e, bool hl, size_t lp)
      : wave(std::move(w)), index(s), start_point(s), end_point(e), has_loop(hl), loop_point(lp) { assert(end_point <= wave->size()); }
  int inputs() const override { return 0; } int outputs() const override { return 1; }
  uint64_t id() const override { return 65; }
  void reset() override { index = start_point; }
  void tick(const float*, float* out) override {
    if (index < end_point) {
      out[0] = (*wave)[index];
      index += 1;
      if (index == end_point && has_loop) index = loop_point;
    } else out[0] = 0.0f;
  }
  FO_CLONE(WavePlayer)
};
// ---- src/resample.rs:210-300 Resample<X> (ID 69): cubic-interpolated variable-speed playback of a generator; input = speed
struct Resample : Node {
  Child x; std::vector<float> buffer; double consumer = 1.0; size_t producer = 0;
  explicit Resample(Node* x_) : x(x_) {
    assert(x->inputs() == 0);
    x->set_sample_rate(DEFAULT_SR);
    AttoHash h = x->ping(true, AttoHash(69)); x->ping(false, h);
    buffer.assign((size_t)x->outputs() * 128, 0.0f);
  }
  int inputs() const override { return 1; } int outputs() const override { return x->outputs(); }
  uint64_t id() const override { return 69; }
  void reset() override { x->reset(); consumer = 1.0; producer = 0; }
  void set_sample_rate(double sr) override { x->set_sample_rate(sr); }
  void tick(const float* in, float* out) override {
    consumer += (double)fmaxf(0.0f, in[0]);
    const double d = consumer - floor(consumer);
    const size_t ci = (size_t)(consumer - d);
    const int no = x->outputs();
    while (ci + 2 >= producer) {
      float inner[256];
      x->tick(nullptr, inner);
      for (int c = 0; c < no; c++) buffer[(size_t)c * 128 + (producer & 0x7f)] = inner[c];
      producer += 1;
    }
    for (int c = 0; c < no; c++) {
      const float* b = &buffer[(size_t)c * 128];
      out[c] = splinef(b[(ci + 0x7f) & 0x7f], b[ci & 0x7f], b[(ci + 1) & 0x7f], b[(ci + 2) & 0x7f], (float)d);
    }
  }
  AttoHash ping(bool probe, AttoHash h) override { return x->ping(probe, h.hash(id())); }
  FO_CLONE(Resample)
};

// ---- src/envelope.rs:185-358 EnvelopeIn<f32, E, U1, f32> (ID 53) specialised to the closed-form
// closure of src/adsr.rs:21-70 `adsr_live(attack, decay, sustain, release)`.
struct AdsrLive : Node {
  float attack, decay, sustain, release;
  // closure state (adsr.rs:27-33): `attacked`, Shared attack_start (a) and release_start (b)
  bool attacked = false; float attack_start = 0.0f, release_start = -1.0f;
  // EnvelopeIn state
  float t = 0, t_0 = 0, t_1 = 0; uint64_t t_hash = 0; float value_0 = 0, value_1 = 0, value = 0, value_d = 0;
  float interval, sample_duration = 0; uint64_t hash = 0;
  AdsrLive(float a, float d, float s, float r) : attack(a), decay(d), sustain(s), release(r), interval((float)0.002) {
    set_sample_rate(DEFAULT_SR); reset();
  }
  static float ads(float attack, float decay, float sustain, float time) {
    if (time < attack) return lerpf(0.0f, 1.0f, time / attack);
    float decay_time = time - attack;
    if (decay_time < decay) return lerpf(1.0f, sustain, decay_time / decay);
    return sustain;
  }
  float envelope(float time, float control) {
    if (release_start >= 0.0f && control > 0.0f) { attacked = true; attack_start = time; release_start = -1.0f; }
    else if (release_start < 0.0f && control <= 0.0f) { release_start = time; }
    if (!attacked) return 0.0f;
    float ads_value = ads(attack, decay, sustain, time - attack_start);
    if (release_start < 0.0f) return ads_value;
    return ads_value * clamp01f(delerpf(release_start + release, release_start, time));
  }
  void next_segment(float input) {  // envelope.rs:238-263
    if (t_0 == 0.0f && t_1 == 0.0f) { value_0 = envelope(t_0, input); }
    else { t_0 = t_1; value_0 = value_1; }
    float next_interval = lerpf(0.75f, 1.25f, (float)rnd1(t_hash)) * interval;
    t_1 = t_0 + next_interval;
    value_1 = envelope(t_1, input);
    t_hash = t_hash * 6364136223846793005ull + 1ull;
    float u = delerpf(t_0, t_1, t);
    value = lerpf(value_0, value_1, u);
    float samples = next_interval / sample_duration;
    value_d = (value_1 - value_0) / samples;
  }
  int inputs() const override { return 1; } int outputs() const override { return 1; }
  uint64_t id() const override { return 53; }
  void reset() override { t = 0; t_0 = 0; t_1 = 0; t_hash = hash; }
  void set_sample_rate(double sr) override { sample_duration = (float)(1.0 / sr); }
  void tick(const float* in, float* out) override {  // :297-305
    if (t >= t_1) next_segment(in[0]);
    out[0] = value; value += value_d; t += sample_duration;
  }
  void process(int size, const float* in, float* out) override {  // :307-341
    if (size == 0) return;
    if (t >= t_1) next_segment(in[0]);
    int i = 0;
    while (i < size) {
      size_t segment_samples_left = (size_t)(int64_t)ceilf((t_1 - t) / sample_duration);
      size_t loop_samples = std::min<size_t>((size_t)(size - i), segment_samples_left);
      float v = value, delta = value_d;
      for (size_t o = 0; o < loop_samples; o++) { out[i + o] = v; v += delta; }
      value = v;
      i += (int)loop_samples;
      t += (float)(int64_t)loop_samples * sample_duration;
      if (loop_samples == segment_samples_left && i < size) next_segment(in[i]);
    }
  }
  void set(const Setting& s) override { if (s.kind == P_INTERVAL) interval = s.v[0]; }
  void set_hash(uint64_t h) override { hash = h; t_hash = h; }
  FO_CLONE(AdsrLive)
};

// ---- src/net.rs:73-146, 175-260, 556-820, 834-916, 1187-1286, 1383-1389; src/vertex.rs:16-122,162-170
struct Port { int type; int node; int port; };  // type 0 Zero, 1 Global(port), 2 Local(node, port)
inline float sine_easef(float x);   // (src/math.rs:453-458, defined with the sequencer below)
inline float fade_atf(int fade, float x) { return fade == 0 ? sine_easef(x) : smooth5f(x); }   // Fade::at (src/sequencer.rs:48-55), 0 Power, 1 Smooth
struct Vertex {
  Child unit; std::vector<Port> source; std::vector<float> input, output, tick_in, tick_out;
  bool has_sv = false; int sv_node = 0, sv_port = 0; int unplugged = 0; bool ordered = false;
  // Net::crossfade (src/net.rs:480-504) / src/vertex.rs:35-39,124-245: the unit we are fading into, the one queued behind it, all in f32
  Child next, latest; bool has_next = false, has_latest = false; int next_fade = 1, latest_fade = 1; float next_fade_time = 0.0f, latest_fade_time = 0.0f;
  float fade_phase = 0.0f; std::vector<float> output_tmp, tick_out_tmp;
  int outs() const { return unit->outputs(); }
  void enqueue(Node* u, int fade, float fade_time) {   // vertex.rs:232-245
    if (has_next) { latest = Child(u); has_latest = true; latest_fade = fade; latest_fade_time = fade_time; }   // replaces a queued unit
    else { next = Child(u); has_next = true; next_fade = fade; next_fade_time = fade_time; fade_phase = 0.0f; }
  }
  void next_phase() {   // vertex.rs:124-135: the faded-in unit becomes the unit; the queued one (if any) starts fading in
    unit = std::move(next);
    next_fade = latest_fade; fade_phase = 0.0f; next_fade_time = latest_fade_time;
    next = std::move(latest); has_next = has_latest; has_latest = false;
  }
  void tick(float sample_rate) {   // vertex.rs:138-160
    unit->tick(tick_in.data(), tick_out.data());
    if (has_next) {
      const int no = outs();
      if ((int)tick_out_tmp.size() < std::max(1, no)) tick_out_tmp.assign(std::max(1, no), 0.0f);
      float f = fade_atf(next_fade, 1.0f - fade_phase);
      for (int c = 0; c < no; c++) tick_out[c] *= f;
      next->tick(tick_in.data(), tick_out_tmp.data());
      f = fade_atf(next_fade, fade_phase);
      for (int c = 0; c < no; c++) tick_out[c] += tick_out_tmp[c] * f;
      fade_phase += 1.0f / (next_fade_time * sample_rate);
      if (fade_phase >= 1.0f) next_phase();
    }
  }
  void process(int size, const float* in, float sample_rate) {   // vertex.rs:163-229
    unit->process(size, in, output.data());
    if (has_next) {
      const int no = outs();
      if (output_tmp.size() < (size_t)std::max(1, no) * B) output_tmp.assign((size_t)std::max(1, no) * B, 0.0f);
      const float pl = (1.0f - fade_phase) * next_fade_time * sample_rate;
      const size_t phase_left = pl != pl || pl <= 0.0f ? 0 : (pl >= 1.8446744073709552e19f ? SIZE_MAX : (size_t)pl);   // `as usize`
      const int n = (int)std::min<size_t>((size_t)size, phase_left);
      const float fade_d = 1.0f / (next_fade_time * sample_rate);
      for (int c = 0; c < no; c++) { float fade = fade_phase; for (int i = 0; i < n; i++) { output[c * B + i] *= fade_atf(next_fade, 1.0f - fade); fade += fade_d; } }
      next->process(size, in, output_tmp.data());
      for (int c = 0; c < no; c++) {
        float fade = fade_phase;
        for (int i = 0; i < n; i++) { output[c * B + i] += output_tmp[c * B + i] * fade_atf(next_fade, fade); fade += fade_d; }
        for (int i = n; i < size; i++) output[c * B + i] = output_tmp[c * B + i];
      }
      fade_phase += (float)n / (next_fade_time * sample_rate);
      if (phase_left <= (size_t)size) next_phase();   // "We don't start fading in the latest unit until the next block."
    }
  }
};
struct Net : Node {
  int nin, nout; std::vector<Port> output_edge; std::vector<Vertex> vertex; std::vector<int> order; bool ordered = false;
  float sample_rate = (float)DEFAULT_SR; bool cycle = false;
  Net(int i, int o) : nin(i), nout(o) { output_edge.assign(o, Port{0, 0, 0}); }
  int inputs() const override { return nin; } int outputs() const override { return nout; }
  uint64_t id() const override { return 63; }
  int push(Node* unit) {
    unit->set_sample_rate((double)sample_rate);
    Vertex v; v.unit = Child(unit);
    v.source.assign(unit->inputs(), Port{0, 0, 0});
    v.input.assign((size_t)std::max(1, unit->inputs()) * B, 0.0f);
    v.output.assign((size_t)std::max(1, unit->outputs()) * B, 0.0f);
    v.tick_in.assign(std::max(1, unit->inputs()), 0.0f); v.tick_out.assign(std::max(1, unit->outputs()), 0.0f);
    vertex.push_back(std::move(v)); ordered = false;
    return (int)vertex.size() - 1;
  }
  void crossfade(int node, int fade, float fade_time, Node* unit) {   // src/net.rs:480-504 (no backend: enqueued at once)
    assert(unit->inputs() == vertex[node].unit->inputs() && unit->outputs() == vertex[node].unit->outputs());
    unit->set_sample_rate((double)sample_rate);
    vertex[node].enqueue(unit, fade, fade_time);
  }
  void connect(int s, int sp, int t, int tp) { assert(s != t); vertex[t].source[tp] = Port{2, s, sp}; ordered = false; }
  void connect_input(int gi, int t, int tp) { vertex[t].source[tp] = Port{1, 0, gi}; ordered = false; }
  void connect_output(int s, int sp, int go) { output_edge[go] = Port{2, s, sp}; ordered = false; }
  void pass_through(int gi, int go) { output_edge[go] = Port{1, 0, gi}; ordered = false; }
  void pipe_input(int t) {
    for (int c = 0; c < vertex[t].unit->inputs(); c++) vertex[t].source[c] = nin > 0 ? Port{1, 0, c % nin} : Port{0, 0, 0};
    ordered = false;
  }
  void pipe_output(int s) {
    int no = vertex[s].unit->outputs();
    for (int c = 0; c < nout; c++) output_edge[c] = no > 0 ? Port{2, s, c % no} : Port{0, 0, 0};
    ordered = false;
  }
  void pipe_all(int s, int t) {
    if (s == t) return;
    int no = vertex[s].unit->outputs();
    for (int c = 0; c < vertex[t].unit->inputs(); c++) vertex[t].source[c] = no > 0 ? Port{2, s, c % no} : Port{0, 0, 0};
    ordered = false;
  }
  int chain(Node* unit) {  // :764-787
    int ui = unit->inputs();
    int idx = push(unit);
    if (vertex.size() == 1) { if (nin > 0) pipe_input(idx); }
    else for (int i = 0; i < ui; i++) vertex[idx].source[i] = nout > 0 ? output_edge[i % nout] : Port{0, 0, 0};
    pipe_output(idx); ordered = false;
    return idx;
  }
  static Net* wrap(Node* unit) {  // :925-935
    Net* n = new Net(unit->inputs(), unit->outputs());
    int id = n->push(unit);
    if (n->nin > 0) n->pipe_input(id);
    if (n->nout > 0) n->pipe_output(id);
    return n;
  }
  void append_vertices(Net& o, int offset, int input_offset, bool global_to_output_edge) {
    for (auto& v : o.vertex) vertex.push_back(v);
    for (size_t node = offset; node < vertex.size(); node++)
      for (auto& s : vertex[node].source) {
        if (s.type == 2) s.node += offset;
        else if (s.type == 1) { if (global_to_output_edge) s = output_edge[s.port]; else s.port += input_offset; }
      }
  }
  // graph algebra (src/net.rs:1447-1832); each consumes both operands and returns a new net (net1 mutated).
  static Net* bus(Net* n1, Net* n2) {
    assert(n1->nin == n2->nin && n1->nout == n2->nout);
    std::vector<Port> o1 = n1->output_edge, o2 = n2->output_edge;
    int offset = (int)n1->vertex.size();
    n1->append_vertices(*n2, offset, 0, false);
    int add_offset = (int)n1->vertex.size();
    for (int i = 0; i < n1->nout; i++) {
      n1->push(new Binop(OP_ADD, new MultiPass(1, true), new MultiPass(1, true)));
      n1->connect_output(add_offset + i, 0, i);
    }
    for (size_t i = 0; i < o1.size(); i++) {
      if (o1[i].type == 2) n1->connect(o1[i].node, o1[i].port, add_offset + (int)i, 0);
      else if (o1[i].type == 1) n1->connect_input(o1[i].port, add_offset + (int)i, 0);
    }
    for (size_t i = 0; i < o2.size(); i++) {
      if (o2[i].type == 2) n1->connect(o2[i].node + offset, o2[i].port, add_offset + (int)i, 1);
      else if (o2[i].type == 1) n1->connect_input(o2[i].port, add_offset + (int)i, 1);
    }
    n1->ordered = false; delete n2; return n1;
  }
  static Net* binary(Net* n1, Net* n2, int op) {
    assert(n1->nout == n2->nout);
    std::vector<Port> o1 = n1->output_edge, o2 = n2->output_edge;
    int input_offset = n1->nin, offset = (int)n1->vertex.size();
    n1->append_vertices(*n2, offset, input_offset, false);
    n1->nin += n2->nin;
    int add_offset = (int)n1->vertex.size();
    for (int i = 0; i < n1->nout; i++) {
      n1->push(new Binop(op, new MultiPass(1, true), new MultiPass(1, true)));
      n1->connect_output(add_offset + i, 0, i);
    }
    for (size_t i = 0; i < o1.size(); i++) {
      if (o1[i].type == 2) n1->connect(o1[i].node, o1[i].port, add_offset + (int)i, 0);
      else if (o1[i].type == 1) n1->connect_input(o1[i].port, add_offset + (int)i, 0);
    }
    for (size_t i = 0; i < o2.size(); i++) {
      if (o2[i].type == 2) n1->connect(o2[i].node + offset, o2[i].port, add_offset + (int)i, 1);
      else if (o2[i].type == 1) n1->connect_input(o2[i].port + input_offset, add_offset + (int)i, 1);
    }
    n1->ordered = false; delete n2; return n1;
  }
  static Net* stack(Net* n1, Net* n2) {
    int offset = (int)n1->vertex.size(), input_offset = n1->nin, output_offset = n1->nout;
    n1->append_vertices(*n2, offset, input_offset, false);
    for (auto e : n2->output_edge) {
      if (e.type == 2) e.node += offset; else if (e.type == 1) e.port += input_offset;
      n1->output_edge.push_back(e);
    }
    (void)output_offset;
    n1->nin += n2->nin; n1->nout += n2->nout;
    n1->ordered = false; delete n2; return n1;
  }
  static Net* branch(Net* n1, Net* n2) {
    assert(n1->nin == n2->nin);
    int offset = (int)n1->vertex.size();
    n1->append_vertices(*n2, offset, 0, false);
    for (auto e : n2->output_edge) { if (e.type == 2) e.node += offset; n1->output_edge.push_back(e); }
    n1->nout += n2->nout;
    n1->ordered = false; delete n2; return n1;
  }
  static Net* pipe(Net* n1, Net* n2) {
    assert(n1->nout == n2->nin);
    int offset = (int)n1->vertex.size();
    n1->append_vertices(*n2, offset, 0, true);
    std::vector<Port> oe1 = n1->output_edge;
    n1->output_edge = n2->output_edge; n1->nout = n2->nout;
    for (auto& e : n1->output_edge) {
      if (e.type == 2) e.node += offset; else if (e.type == 1) e = oe1[e.port];
    }
    n1->ordered = false; delete n2; return n1;
  }
  // ---- ordering (:834-916)
  void determine_order() {
    for (auto& v : vertex) {  // vertex.rs:98-122 update_source_vertex
      v.has_sv = false;
      int ni = v.unit->inputs(); if (ni == 0) continue;
      bool ok = true; int sn = 0, sp = 0;
      for (int i = 0; i < ni && ok; i++) {
        Port s = v.source[i];
        if (s.type == 2) { if (i == 0) { sn = s.node; sp = s.port; } else if (sn != s.node || sp + i != s.port) ok = false; }
        else ok = false;
      }
      if (ok) { v.has_sv = true; v.sv_node = sn; v.sv_port = sp; }
    }
    AttoHash h = ping(true, AttoHash(id())); ping(false, h);
    order.clear();
    for (auto& v : vertex) { v.unplugged = 0; v.ordered = false; }
    for (auto& v : vertex) for (int c = 0; c < v.unit->inputs(); c++) if (v.source[c].type == 2) vertex[v.source[c].node].unplugged += 1;
    for (size_t i = 0; i < vertex.size(); i++) {
      if (vertex[i].ordered) continue;
      if (vertex[i].unplugged == 0) { vertex[i].ordered = true; order.push_back((int)i); propagate((int)i); }
    }
    cycle = order.size() < vertex.size();
    if (cycle) for (size_t i = 0; i < vertex.size(); i++) if (!vertex[i].ordered) order.push_back((int)i);
    std::reverse(order.begin(), order.end());
    ordered = true;
  }
  void propagate(int i) {  // explicit stack instead of recursion, same visiting order as :877-888
    struct Fr { int node; int ch; };
    std::vector<Fr> st; st.push_back({i, 0});
    while (!st.empty()) {
      Fr& f = st.back();
      if (f.ch >= vertex[f.node].unit->inputs()) { st.pop_back(); continue; }
      Port s = vertex[f.node].source[f.ch]; f.ch++;
      if (s.type == 2) {
        int j = s.node;
        vertex[j].unplugged -= 1;
        if (vertex[j].unplugged == 0) { vertex[j].ordered = true; order.push_back(j); st.push_back({j, 0}); }
      }
    }
  }
  void set_sample_rate(double sr) override {
    float s = (float)sr;
    if (sample_rate != s) { sample_rate = s; for (auto& v : vertex) v.unit->set_sample_rate((double)s); if (!ordered) determine_order(); }
  }
  void reset() override { for (auto& v : vertex) v.unit->reset(); if (!ordered) determine_order(); }
  void tick(const float* in, float* out) override {
    if (!ordered) determine_order();
    for (int ni : order) {
      Vertex& v = vertex[ni];
      for (int c = 0; c < v.unit->inputs(); c++) {
        Port s = v.source[c];
        v.tick_in[c] = s.type == 0 ? 0.0f : s.type == 1 ? in[s.port] : vertex[s.node].tick_out[s.port];
      }
      v.tick(sample_rate);
    }
    for (int c = 0; c < nout; c++) {
      Port s = output_edge[c];
      out[c] = s.type == 0 ? 0.0f : s.type == 1 ? in[s.port] : vertex[s.node].tick_out[s.port];
    }
  }
  void process(int size, const float* in, float* out) override {
    if (!ordered) determine_order();
    const int len = simd_items(size) * 8;
    for (int ni : order) {
      Vertex& v = vertex[ni];
      if (v.has_sv) {
        v.process(size, vertex[v.sv_node].output.data() + v.sv_port * B, sample_rate);
      } else {
        for (int c = 0; c < v.unit->inputs(); c++) {
          Port s = v.source[c];
          for (int i = 0; i < len; i++) v.input[c * B + i] = s.type == 0 ? 0.0f : s.type == 1 ? in[s.port * B + i] : vertex[s.node].output[s.port * B + i];
        }
        v.process(size, v.input.data(), sample_rate);
      }
    }
    for (int c = 0; c < nout; c++) {
      Port s = output_edge[c];
      for (int i = 0; i < len; i++) out[c * B + i] = s.type == 0 ? 0.0f : s.type == 1 ? in[s.port * B + i] : vertex[s.node].output[s.port * B + i];
    }
  }
  void set(const Setting& s) override {
    Address d = s.direction();
    if (d.type == 2 && d.value < vertex.size()) vertex[d.value].unit->set(s.peel());
  }
  AttoHash ping(bool probe, AttoHash h) override {
    h = h.hash(id());
    for (auto& v : vertex) h = v.unit->ping(probe, h);
    return h;
  }
  FO_CLONE(Net)
};

// ---- src/sequencer.rs Sequencer (ID 64) without a backend: sample-accurate start / stop of units with fade envelopes.
// Restated in full for ReplayMode::None / All / Loop(t), tick (:679-751) and process (:753-873), including the block-relative fade
// indices applied to the unit's own buffer (:113-217) and BufferRef::span as written (src/buffer.rs:216-222: it copies input[start]
// to every slot and only when length > start). std's BinaryHeap is restated from liballoc (push = sift_up with a strict compare,
// pop = swap with the last, sift_down_to_bottom preferring the right child on ties, sift_up): ONLY the order in which events with
// identical start times become active depends on it, i.e. the association order of their f32 sum.
inline float sine_easef(float x) {   // src/math.rs:453-458, T = f32
  x = x * (float)(3.141592653589793 * 0.5);
  return 16.0f * x * ((float)3.141592653589793 - x) / ((float)(5.0 * 3.141592653589793 * 3.141592653589793) - 4.0f * x * ((float)3.141592653589793 - x));
}
inline double round_away(double x) { return round(x); }              // f64::round: half away from zero
inline size_t as_usize(double x) { return x != x || x <= 0.0 ? 0 : (x >= 1.8446744073709552e19 ? SIZE_MAX : (size_t)x); }   // saturating `as usize`
struct SeqEvent {
  Child unit; double start_time, end_time, original_start_time, original_end_time; int fade_ease; double fade_in, fade_out; uint64_t id;
};
struct Sequencer : Node {
  enum Mode { ALL = 0, NONE = 1, LOOP = 2 };
  struct Edit { double end_time, fade_out; };
  std::vector<SeqEvent> active, ready /* binary heap, earliest start at the root */, past;
  std::map<uint64_t, size_t> active_map; std::map<uint64_t, Edit> edit_map;
  double active_threshold = 0.0; int nin, nout; double time = 0.0, sample_rate = DEFAULT_SR, sample_duration = 1.0 / DEFAULT_SR;
  std::vector<float> buffer, tick_buffer, input_buffer; int mode; double loop_arg, loop_point = 0.0; uint64_t next_id = 1;
  Sequencer(int i, int o, int mode_, double loop_t) : nin(i), nout(o), mode(mode_), loop_arg(loop_t) {
    buffer.assign((size_t)std::max(1, o) * B, 0.0f); tick_buffer.assign(std::max(1, o), 0.0f); input_buffer.assign((size_t)std::max(1, i) * B, 0.0f);
    reset();
  }
  bool is_replay() const { return mode != NONE; } bool is_loop() const { return mode == LOOP; }
  // BinaryHeap<Event> with Ord reversed on start_time (total_cmp): a <= b in heap order  <=>  a.start >= b.start
  static bool heap_le(const SeqEvent& a, const SeqEvent& b) { return !(a.start_time < b.start_time); }
  void heap_sift_up(size_t start, size_t pos) {
    SeqEvent hole = std::move(ready[pos]);
    while (pos > start) { size_t parent = (pos - 1) / 2; if (heap_le(hole, ready[parent])) break; ready[pos] = std::move(ready[parent]); pos = parent; }
    ready[pos] = std::move(hole);
  }
  void heap_push(SeqEvent e) { ready.push_back(std::move(e)); heap_sift_up(0, ready.size() - 1); }
  SeqEvent heap_pop() {
    SeqEvent item = std::move(ready.back()); ready.pop_back();
    if (!ready.empty()) {
      std::swap(item, ready[0]);
      const size_t end = ready.size(); size_t pos = 0;
      SeqEvent hole = std::move(ready[0]);
      size_t child = 1;
      while (child <= (end >= 2 ? end - 2 : 0)) {   // end.saturating_sub(2)
        if (heap_le(ready[child], ready[child + 1])) child += 1;
        ready[pos] = std::move(ready[child]); pos = child; child = 2 * pos + 1;
      }
      if (child == end - 1) { ready[pos] = std::move(ready[child]); pos = child; }
      ready[pos] = std::move(hole);
      heap_sift_up(0, pos);
    }
    return item;
  }
  int inputs() const override { return nin; } int outputs() const override { return nout; }
  uint64_t id() const override { return 64; }
  uint64_t push(double start, double end, int ease, double fin, double fout, Node* unit) {   // :319-345
    assert(unit->inputs() == nin && unit->outputs() == nout);
    const double duration = end - start; assert(fin <= duration && fout <= duration); (void)duration;
    unit->set_sample_rate(sample_rate);
    SeqEvent e{Child(unit), start, end, start, end, ease, fin, fout, next_id++};
    const uint64_t eid = e.id; push_event(std::move(e)); return eid;
  }
  void push_event(SeqEvent e) {   // :347-360
    if (e.start_time < active_threshold) { active_map[e.id] = active.size(); active.push_back(std::move(e)); } else heap_push(std::move(e));
  }
  uint64_t push_relative(double start, double end, int ease, double fin, double fout, Node* unit) {   // :376-418
    unit->set_sample_rate(sample_rate);
    SeqEvent e{Child(unit), start + time, end + time, start, end, ease, fin, fout, next_id++};
    e.original_start_time = start; e.original_end_time = end;   // Event::new ran before the shift (:392-400)
    const uint64_t eid = e.id; push_event(std::move(e)); return eid;
  }
  void edit(uint64_t eid, double end_time, double fade_out) {   // :441-483
    auto it = active_map.find(eid);
    if (it != active_map.end()) {
      SeqEvent& e = active[it->second];
      e.original_end_time = end_time; e.end_time = end_time + e.start_time - e.original_start_time; e.fade_out = fade_out;
    } else if (end_time < active_threshold) { if (is_replay()) edit_map[eid] = Edit{end_time, fade_out}; }
    else edit_map[eid] = Edit{end_time, fade_out};
  }
  void edit_relative(uint64_t eid, double end_time, double fade_out) {   // :486-528
    auto it = active_map.find(eid);
    if (it != active_map.end()) {
      SeqEvent& e = active[it->second];
      e.end_time = time + end_time; e.original_end_time = e.end_time + e.original_start_time - e.start_time; e.fade_out = fade_out;
    } else if (time + end_time < active_threshold) { if (is_replay()) edit_map[eid] = Edit{time + end_time, fade_out}; }
    else edit_map[eid] = Edit{time + end_time, fade_out};
  }
  void ready_to_active(double next_end_time) {   // :531-553
    active_threshold = next_end_time - sample_duration * 0.5;
    while (!ready.empty() && ready[0].start_time < active_threshold) {
      SeqEvent e = heap_pop();
      active_map[e.id] = active.size();
      auto ed = edit_map.find(e.id);
      if (ed != edit_map.end()) { e.fade_out = ed->second.fade_out; e.end_time = ed->second.end_time; edit_map.erase(ed); }
      active.push_back(std::move(e));
    }
  }
  void end_of_event(size_t i) {   // :622-639
    active_map.erase(active[i].id);
    if (i + 1 < active.size()) active_map[active.back().id] = i;
    SeqEvent e = std::move(active[i]);
    if (i + 1 < active.size()) active[i] = std::move(active.back());
    active.pop_back();
    e.start_time = e.original_start_time; e.end_time = e.original_end_time;
    if (is_replay()) e.unit->reset();
    if (is_loop() && e.start_time >= time) heap_push(std::move(e)); else past.push_back(std::move(e));
  }
  void reset() override {   // :642-683
    loop_point = is_loop() ? fmax(64.0 * sample_duration, round_away(loop_arg * sample_rate) / sample_rate) : INFINITY;
    if (mode == NONE) { ready.clear(); past.clear(); active.clear(); edit_map.clear(); active_map.clear(); }
    else {
      if (is_loop()) { for (auto& e : active) { e.start_time -= loop_point; e.end_time -= loop_point; } }
      else { while (!active.empty()) { SeqEvent e = std::move(active.back()); active.pop_back(); e.unit->reset(); heap_push(std::move(e)); } active_map.clear(); }
      while (!past.empty()) { SeqEvent e = std::move(past.back()); past.pop_back(); heap_push(std::move(e)); }
    }
    time = 0.0; active_threshold = 0.0;
  }
  void set_sample_rate(double sr) override {   // :685-701
    if (sample_rate != sr) {
      sample_rate = sr; sample_duration = 1.0 / sr;
      while (!ready.empty()) { SeqEvent e = heap_pop(); e.unit->set_sample_rate(sr); active.push_back(std::move(e)); }
      for (auto& e : past) e.unit->set_sample_rate(sr);
      for (auto& e : active) e.unit->set_sample_rate(sr);
      reset();
    }
  }
  static float ease(int kind, float x) { return kind == 0 ? sine_easef(x) : smooth5f(x); }   // Fade::Power = 0, Fade::Smooth = 1
  void tick(const float* in, float* out) override {   // :704-766
    if (!is_replay()) past.clear();
    for (int c = 0; c < nout; c++) out[c] = 0.0f;
    const double end_time = time + sample_duration;
    ready_to_active(end_time);
    size_t i = 0;
    while (i < active.size()) {
      if (active[i].end_time <= time + 0.5 * sample_duration) end_of_event(i);
      else {
        SeqEvent& e = active[i];
        e.unit->tick(in, tick_buffer.data());
        if (e.fade_in > 0.0) {
          const float f = (float)((time - e.start_time) / ((e.start_time + e.fade_in) - e.start_time));
          if (f < 1.0f) for (int c = 0; c < nout; c++) tick_buffer[c] *= ease(e.fade_ease, f);
        }
        if (e.fade_out > 0.0) {
          const float f = (float)((time - (e.end_time - e.fade_out)) / (e.end_time - (e.end_time - e.fade_out)));
          if (f > 0.0f) for (int c = 0; c < nout; c++) tick_buffer[c] *= ease(e.fade_ease, 1.0f - f);
        }
        for (int c = 0; c < nout; c++) out[c] += tick_buffer[c];
        i += 1;
      }
    }
    time = end_time;
    if (time + 0.5 * sample_duration >= loop_point) reset();
  }
  void process(int size_, const float* in, float* out) override {   // :768-873
    if (!is_replay()) past.clear();
    if (size_ == 0) return;
    const size_t size = (size_t)size_;
    for (int c = 0; c < nout; c++) for (int j = 0; j < B; j++) out[c * B + j] = 0.0f;
    const double end_time = fmin(time + sample_duration * (double)size, loop_point);
    ready_to_active(end_time);
    const size_t loop_size = is_loop() ? as_usize(round_away(fmax(0.0, loop_point - time) * sample_rate)) : size;
    size_t i = 0;
    while (i < active.size()) {
      if (active[i].end_time <= time + 0.5 * sample_duration) { end_of_event(i); continue; }
      SeqEvent& e = active[i];
      const size_t start_index = e.start_time <= time ? 0 : as_usize(round_away((e.start_time - time) * sample_rate));
      const size_t end_index = e.end_time >= end_time ? std::min(size, loop_size) : std::min(loop_size, as_usize(round_away((e.end_time - time) * sample_rate)));
      if (end_index > start_index) {
        const float* node_input = in;
        if (start_index != 0) {   // input.span(start_index, end_index - start_index, &mut input_buffer) as written
          for (int c = 0; c < nin; c++) for (size_t k = start_index; k < end_index - start_index; k++) input_buffer[c * B + (k - start_index)] = in[c * B + start_index];
          node_input = input_buffer.data();
        }
        e.unit->process((int)(end_index - start_index), node_input, buffer.data());
        {   // fade_in :113-160
          const double fade_duration = e.fade_in, fade_start_time = e.start_time, fade_end_time = fade_start_time + fade_duration;
          if (fade_duration > 0.0 && fade_end_time > time) {
            const size_t fade_end_i = fade_end_time >= end_time ? end_index : as_usize(round_away((fade_end_time - time) / sample_duration));
            const float fade_phase = (float)(((time + (double)start_index * sample_duration) - fade_start_time) / (fade_end_time - fade_start_time));
            const float fade_d = (float)(sample_duration / fade_duration);
            for (int c = 0; c < nout; c++) { float fade = fade_phase; for (size_t k = 0; k < fade_end_i; k++) { buffer[c * B + k] *= ease(e.fade_ease, fade); fade += fade_d; } }
          }
        }
        {   // fade_out :162-217
          const double fade_duration = e.fade_out, fade_end_time = e.end_time, fade_start_time = fade_end_time - fade_duration;
          if (fade_duration > 0.0 && fade_start_time < end_time) {
            const size_t fade_i = fade_start_time <= time ? 0 : as_usize(round_away((fade_start_time - time) / sample_duration));
            const float fade_phase = (float)(((time + (double)fade_i * sample_duration) - fade_start_time) / (fade_end_time - fade_start_time));
            const float fade_d = (float)(sample_duration / fade_duration);
            for (int c = 0; c < nout; c++) { float fade = fade_phase; for (size_t k = fade_i; k < end_index; k++) { buffer[c * B + k] *= ease(e.fade_ease, 1.0f - fade); fade += fade_d; } }
          }
        }
        for (int c = 0; c < nout; c++) for (size_t j = start_index; j < end_index; j++) out[c * B + j] += buffer[c * B + (j - start_index)];
      }
      i += 1;
    }
    time = end_time;
    if (loop_size < size) {   // wrap around the loop point and render the rest of the block (:845-872)
      reset();
      // As written, both copy loops run `for j in loop_size - size..size`: with loop_size < size the start wraps (release builds; a
      // debug build panics on the subtraction) and the ranges are empty, so the remainder is rendered from a zero input into a
      // scratch buffer and the block's tail stays silent. Restated as written.
      std::vector<float> lin((size_t)std::max(1, nin) * B, 0.0f), lout((size_t)std::max(1, nout) * B, 0.0f);
      process((int)(size - loop_size), lin.data(), lout.data());
    }
  }
  Node* clone() const override {
    Sequencer* s = new Sequencer(nin, nout, mode, loop_arg);
    s->active = active; s->ready = ready; s->past = past; s->active_map = active_map; s->edit_map = edit_map; s->active_threshold = active_threshold;
    s->time = time; s->sample_rate = sample_rate; s->sample_duration = sample_duration; s->loop_point = loop_point; s->next_id = next_id;
    return s;
  }
};

// ---- src/slot.rs Slot + SlotBackend (ID 78) merged: a unit that can be replaced with a crossfade. `set` queues an update that the
// next tick / process picks up (handle_messages :124-142): the first becomes `next` and fades in over fade_time while `current` fades
// out; one that arrives during a fade waits as `latest` (replacing an earlier one) and starts when the fade ends. Units are NOT re-rated
// on arrival (only set_sample_rate touches them, :175-185).
struct Slot : Node {
  struct Update { int fade; double fade_time; Child unit; };
  int nin, nout; double sample_rate = DEFAULT_SR;
  Child current, next, latest; bool has_next = false, has_latest = false;
  int fade = 1, latest_fade = 1; double fade_time = 0.0, fade_phase = 0.0, latest_fade_time = 0.0;
  std::vector<Update> queue; std::vector<float> buffer, tick_buf;
  explicit Slot(Node* unit) : nin(unit->inputs()), nout(unit->outputs()), current(unit) {
    current->set_sample_rate(DEFAULT_SR);
    buffer.assign((size_t)std::max(1, nout) * B, 0.0f); tick_buf.assign(std::max(1, nout), 0.0f);
  }
  void set(int fade_, double fade_time_, Node* unit) { assert(unit->inputs() == nin && unit->outputs() == nout); queue.push_back(Update{fade_, fade_time_, Child(unit)}); }
  void handle_messages() {
    for (auto& m : queue) {
      if (!has_next) { next = std::move(m.unit); has_next = true; fade_phase = 0.0; fade_time = m.fade_time; fade = m.fade; }
      else { latest = std::move(m.unit); has_latest = true; latest_fade = m.fade; latest_fade_time = m.fade_time; }
    }
    queue.clear();
  }
  void next_phase() {   // :143-151
    current = std::move(next);
    fade = latest_fade; fade_phase = 0.0; fade_time = latest_fade_time;
    if (has_latest) { next = std::move(latest); has_next = true; has_latest = false; } else has_next = false;
  }
  int inputs() const override { return nin; } int outputs() const override { return nout; }
  uint64_t id() const override { return 78; }
  void reset() override {   // :156-172: adopt the latest configuration, then reset it
    if (has_latest) { current = std::move(latest); has_latest = false; has_next = false; }
    else if (has_next) { current = std::move(next); has_next = false; }
    current->reset();
  }
  void set_sample_rate(double sr) override {
    sample_rate = sr; current->set_sample_rate(sr);
    if (has_next) next->set_sample_rate(sr);
    if (has_latest) latest->set_sample_rate(sr);
  }
  static float ease(int kind, float x) { return kind == 0 ? sine_easef(x) : smooth5f(x); }
  void tick(const float* in, float* out) override {   // :187-203
    handle_messages();
    current->tick(in, out);
    if (has_next) {
      const float f = (float)ease_d(fade, 1.0 - fade_phase);
      for (int c = 0; c < nout; c++) out[c] *= f;
      next->tick(in, tick_buf.data());
      const float g = (float)ease_d(fade, fade_phase);
      for (int c = 0; c < nout; c++) out[c] += tick_buf[c] * g;
      fade_phase += 1.0 / (fade_time * sample_rate);
      if (fade_phase >= 1.0) next_phase();
    }
  }
  static double ease_d(int kind, double x) {   // Fade::at::<f64> on the tick path
    if (kind == 1) return ((x * 6.0 - 15.0) * x + 10.0) * x * x * x;
    const double PI = 3.141592653589793; x = x * (PI * 0.5);
    return 16.0 * x * (PI - x) / (5.0 * PI * PI - 4.0 * x * (PI - x));
  }
  void process(int size_, const float* in, float* out) override {   // :205-262
    handle_messages();
    const size_t size = (size_t)size_;
    current->process(size_, in, out);
    if (has_next) {
      const size_t phase_left = as_usize((1.0 - fade_phase) * fade_time * sample_rate);
      const size_t n = std::min(size, phase_left);
      const float fade_d = (float)(1.0 / (fade_time * sample_rate));
      for (int c = 0; c < nout; c++) { float f = (float)fade_phase; for (size_t i = 0; i < n; i++) { out[c * B + i] *= ease(fade, 1.0f - f); f += fade_d; } }
      next->process(size_, in, buffer.data());
      for (int c = 0; c < nout; c++) {
        float f = (float)fade_phase;
        for (size_t i = 0; i < n; i++) { out[c * B + i] += buffer[c * B + i] * ease(fade, f); f += fade_d; }
        for (size_t i = n; i < size; i++) out[c * B + i] = buffer[c * B + i];
      }
      fade_phase += (double)n / (fade_time * sample_rate);
      if (phase_left <= size) next_phase();
    }
  }
  AttoHash ping(bool probe, AttoHash h) override { (void)probe; return h.hash(id()); }   // set_hash on the boxed units reaches leaves only (:279-291)
  Node* clone() const override {
    Slot* s2 = new Slot(current->clone());
    s2->sample_rate = sample_rate; s2->has_next = has_next; s2->has_latest = has_latest; if (has_next) s2->next = next; if (has_latest) s2->latest = latest;
    s2->fade = fade; s2->latest_fade = latest_fade; s2->fade_time = fade_time; s2->fade_phase = fade_phase; s2->latest_fade_time = latest_fade_time; s2->queue = queue;
    return s2;
  }
};

}  // namespace fo
