// workers.h — the host threads of the drivers: child contexts for vsg_search_batch / vsg_allpairs (search.cu) and one
// thread per device or per child for them and for the multi-GPU entry points (group.cu).
#pragma once

#include "vsg_internal.h"

#include <algorithm>
#include <string>
#include <thread>
#include <vector>

namespace vsg {

// c's first n child contexts (created as needed), one per host thread: c's scoring and kernel choices, and an
// equal share of its direction-bit budget
inline int prepare_children(vsg_ctx * c, int n)
{
  while (static_cast<int>(c->children.size()) < n) {
    vsg_ctx * ch = nullptr;
    int const r = vsg_ctx_create(c->device, &c->scoring, &ch);
    if (r != VSG_OK) { return r; }
    c->children.push_back(ch);
  }
  for (int t = 0; t < n; t++) {
    vsg_ctx * ch = c->children[static_cast<size_t>(t)];
    ch->dir_budget = std::max<size_t>(c->dir_budget / static_cast<size_t>(n), static_cast<size_t>(1) << 30);
    ch->fast_disabled = c->fast_disabled;
    ch->ckpt_enabled = c->ckpt_enabled;
  }
  return VSG_OK;
}

// adds the profile of c's first n children to c's own and resets theirs
inline void absorb_children(vsg_ctx * c, int n)
{
  for (int t = 0; t < n; t++) {
    vsg_ctx * ch = c->children[static_cast<size_t>(t)];
    c->prof_cells += ch->prof_cells; c->prof_fast += ch->prof_fast; c->prof_exact += ch->prof_exact;
    c->prof_tb_skipped += ch->prof_tb_skipped; c->prof_tb_redone += ch->prof_tb_redone;
    c->prof_fwd_launches += ch->prof_fwd_launches;
    c->prof_fwd_ms += ch->prof_fwd_ms; c->prof_tb_ms += ch->prof_tb_ms; c->prof_rank_ms += ch->prof_rank_ms;
    vsg_profile_reset(ch);
  }
}

// fn(i) -> VSG_* for every i in [0, n), each on its own thread (on the calling thread when n == 1).  The error
// message lives per thread, so each failure's is kept; the lowest failing i's code and message are returned.
template <class Fn>
int run_parallel(int n, Fn && fn)
{
  std::vector<int> rcs(static_cast<size_t>(n), VSG_OK);
  std::vector<std::string> msgs(static_cast<size_t>(n));
  auto one = [&](int i) {
    int const r = fn(i);
    if (r != VSG_OK) { rcs[static_cast<size_t>(i)] = r; msgs[static_cast<size_t>(i)] = vsg_last_error(); }
  };
  if (n == 1) {
    one(0);
  } else {
    std::vector<std::thread> pool;
    for (int i = 0; i < n; i++) { pool.emplace_back(one, i); }
    for (auto & th : pool) { th.join(); }
  }
  for (int i = 0; i < n; i++) {
    if (rcs[static_cast<size_t>(i)] != VSG_OK) { Error::set(msgs[static_cast<size_t>(i)]); return rcs[static_cast<size_t>(i)]; }
  }
  return VSG_OK;
}

}  // namespace vsg
