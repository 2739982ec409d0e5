// C entry points over the reference's OWN samplers and partitioners -- test infrastructure.
// oracle/Makefile compiles this file together with the reference's scanner/engine/sampler.cpp (unmodified) into
// oracle/_ref/libref_sampler.so; tests/test_reference_samplers_cpu.py compares the engine's Sample / Space / Slice
// row algebra with it on random arguments.  Interfaces used: DomainSampler (sampler.h:36-63), Partitioner (:75-103),
// make_domain_sampler_instance (:66-69), make_partitioner_instance (:105-107).
#include <cstring>
#include <memory>

#include "scanner/engine/sampler.h"

using scanner::Result;
using scanner::i64;
using scanner::u8;
namespace si = scanner::internal;

static int fail(const Result& r, char* err, size_t cap) {
  if (err && cap) {
    strncpy(err, r.msg().c_str(), cap - 1);
    err[cap - 1] = 0;
  }
  return -1;
}

// Rows of the sampled stream over an input of num_upstream rows: out_rows[k] = downstream row id,
// out_map[k] = the upstream row it is (or -1 for a null row).  Returns the count, -1 on error (message in err),
// -2 if cap is too small.  *num_downstream = get_num_downstream_rows(num_upstream).
extern "C" long ref_sampler_downstream(const char* type, const unsigned char* args, size_t n_args, long num_upstream,
                                        long* out_rows, long* out_map, size_t cap, long* num_downstream, char* err,
                                        size_t err_cap) {
  si::DomainSampler* raw = nullptr;
  Result r = si::make_domain_sampler_instance(type, std::vector<u8>(args, args + n_args), raw);
  if (!r.success()) return fail(r, err, err_cap);
  std::unique_ptr<si::DomainSampler> s(raw);
  i64 nd = 0;
  r = s->get_num_downstream_rows(num_upstream, nd);
  if (!r.success()) return fail(r, err, err_cap);
  *num_downstream = nd;
  // the way the reference's analysis uses a sampler (dag_analysis.cpp): the rows wanted downstream name the
  // upstream rows they need, and those rows are then mapped back
  std::vector<i64> want((size_t)nd), up, down, map;
  for (i64 i = 0; i < nd; ++i) want[(size_t)i] = i;
  r = s->get_upstream_rows(want, up);
  if (!r.success()) return fail(r, err, err_cap);
  r = s->get_downstream_rows(up, down, map);
  if (!r.success()) return fail(r, err, err_cap);
  if (down.size() > cap) return -2;
  for (size_t k = 0; k < down.size(); ++k) {
    out_rows[k] = down[k];
    out_map[k] = map[k] < 0 ? -1 : up[(size_t)map[k]];
  }
  return (long)down.size();
}

// Upstream rows needed for the given downstream rows (what derive_stencil_requirements asks a sampler).
extern "C" long ref_sampler_upstream(const char* type, const unsigned char* args, size_t n_args, const long* downstream,
                                      size_t n_down, long* out, size_t cap, char* err, size_t err_cap) {
  si::DomainSampler* raw = nullptr;
  Result r = si::make_domain_sampler_instance(type, std::vector<u8>(args, args + n_args), raw);
  if (!r.success()) return fail(r, err, err_cap);
  std::unique_ptr<si::DomainSampler> s(raw);
  std::vector<i64> down(downstream, downstream + n_down), up;
  r = s->get_upstream_rows(down, up);
  if (!r.success()) return fail(r, err, err_cap);
  if (up.size() > cap) return -2;
  for (size_t k = 0; k < up.size(); ++k) out[k] = up[k];
  return (long)up.size();
}

// Groups of a partitioner over num_rows rows: rows of all groups concatenated in out_rows, group g = out_rows[offsets[g]
// .. offsets[g + 1]).  Returns the number of groups.
extern "C" long ref_partitioner_groups(const char* type, const unsigned char* args, size_t n_args, long num_rows,
                                        long* out_rows, size_t cap, long* offsets, size_t off_cap, char* err,
                                        size_t err_cap) {
  si::Partitioner* raw = nullptr;
  Result r = si::make_partitioner_instance(type, std::vector<u8>(args, args + n_args), num_rows, raw);
  if (!r.success()) return fail(r, err, err_cap);
  std::unique_ptr<si::Partitioner> p(raw);
  const i64 groups = p->total_groups();
  if ((size_t)groups + 1 > off_cap) return -2;
  size_t n = 0;
  for (i64 g = 0; g < groups; ++g) {
    offsets[g] = (long)n;
    const si::PartitionGroup pg = p->group_at(g);
    if (n + pg.rows.size() > cap) return -2;
    for (i64 row : pg.rows) out_rows[n++] = row;
  }
  offsets[groups] = (long)n;
  return (long)groups;
}
