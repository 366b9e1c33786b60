/* oracle/seam2_cluster_strand_driver.cpp — TEST INFRASTRUCTURE ONLY.
 *
 * seam2_cluster_driver.cpp with --strand both (Parameters::opt_strand) set: the same keys, the same records.  Linked
 * twice by oracle/strand.mk, against the UNMODIFIED reference and against shim/cluster_session_vsg.cpp (+ libvsg.so),
 * so that tests/test_cluster_strand_gpu.py can diff the two.  The driver's own source is compiled here unchanged; its
 * one call to vsearch_session_begin() is routed through begin_both_strands(), which sets the option first.
 *
 *   seam2_cluster_strand_driver reads.fasta [key=value ...]
 */
#include "vsearch_api.h"
#include "core/mask.hpp"

namespace {
auto begin_both_strands(struct Parameters & p) -> void
{
  p.opt_strand = true;
  vsearch_session_begin(p);
}
}  // namespace

#define vsearch_session_begin begin_both_strands
#include "seam2_cluster_driver.cpp"
