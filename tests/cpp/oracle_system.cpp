// TEST INFRASTRUCTURE: System<X, F> (src/system.rs:14-97, ID 67) restated on the oracle's nodes, for the tests of `update`. It is built
// by tests/update_oracle.py into a library of its own next to the oracle's; its System takes any oracle node as X (handles of either
// library are fo::Node*). The update function is the oracle's closure interpreter (oracle/fo_closure.h) evaluating the arguments of the
// function's `set` statements, which are then applied in order through the oracle nodes' own set().
#include "../../oracle/fo_closure.h"

using namespace fo;

#define API extern "C" __attribute__((visibility("default")))

struct UpdateSet { int kind, nargs; std::vector<uint64_t> address; };

struct System : Node {
  Child x; cl::Closure f; std::vector<UpdateSet> sets; int nargs;
  float time = 0.0f, delta_time = 0.0f, update_interval, sample_rate = (float)44100.0;   // DEFAULT_SR as f32
  System(Node* x_, float dt, cl::Closure c, std::vector<UpdateSet> s, int na) : x(x_), f(std::move(c)), sets(std::move(s)), nargs(na), update_interval(dt) {
    ctor_ping();   // System::new: ping(true, AttoHash::new(ID)) then ping(false, hash), through System::ping
  }
  int inputs() const override { return x.p->inputs(); }
  int outputs() const override { return x.p->outputs(); }
  uint64_t id() const override { return 67; }
  void reset() override { x.p->reset(); time = 0.0f; delta_time = 0.0f; }
  void set_sample_rate(double sr) override { x.p->set_sample_rate(sr); sample_rate = (float)sr; }
  // (self.f)(self.time, self.delta_time, &mut self.x): the arguments of every statement, then each set in order
  void update() {
    std::vector<float> a((size_t)nargs + 1, 0.0f);
    const float dt[2] = {delta_time, 0.0f};
    f.call(dt, time, a.data());
    int k = 0;
    for (const UpdateSet& u : sets) {
      Setting s; s.kind = u.kind;
      for (int j = 0; j < u.nargs; j++) s.v[j] = a[(size_t)k + j];
      k += u.nargs;
      for (uint64_t v : u.address) s.address.push_back(Address{1, v});
      x.p->set(s);
    }
  }
  void tick(const float* in, float* out) override {
    const float delta_now = 1.0f / sample_rate;
    if (delta_time >= update_interval || time == 0.0f) { update(); delta_time = 0.0f; }
    time += delta_now;
    delta_time += delta_now;
    x.p->tick(in, out);
  }
  void process(int size, const float* in, float* out) override {
    const float delta_now = (float)size / sample_rate;
    if (delta_time >= update_interval || (time == 0.0f && size > 0)) { update(); delta_time = 0.0f; }
    time += delta_now;
    delta_time += delta_now;
    x.p->process(size, in, out);
  }
  void set(const Setting& s) override { x.p->set(s); }
  AttoHash ping(bool probe, AttoHash hash) override { return x.p->ping(probe, hash.hash(id())); }
  FO_CLONE(System)
};

// `text`: |t, dt, _| whose value is the tuple of every statement's arguments in order (tests/update_oracle.py writes it from the update
// text); statement k has kinds[k], nargs[k] arguments and naddr[k] Index steps, all concatenated in addr. Consumes x; null when the
// text does not parse.
API Node* fos_system(Node* x, float dt, const char* text, int ncaps, const char* const* names, const float* values, int nsets, const int* kinds,
                     const int* nargs, const int* naddr, const int64_t* addr) {
  cl::Closure c;
  if (!c.parse(text, 2, 2, ncaps, names, values)) { delete x; return nullptr; }
  std::vector<UpdateSet> sets;
  int total = 0;
  for (int k = 0; k < nsets; k++) {
    UpdateSet u{kinds[k], nargs[k], {}};
    for (int j = 0; j < naddr[k]; j++) u.address.push_back((uint64_t)*addr++);
    total += nargs[k];
    sets.push_back(std::move(u));
  }
  return new System(x, dt, std::move(c), std::move(sets), total);
}
