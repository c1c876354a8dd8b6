// ORACLE — TEST INFRASTRUCTURE ONLY (see requirements.h header). Consolidation validation on top of the oracle's Solve,
// candidate ranking and consolidation probes (oracle.h). Built into _build/libvalidation_oracle.so by validation.mk,
// linked to liboracle.so, so fast mode (oracle_set_fast) covers it too.
#pragma once
#include <string>
#include <utility>
#include <vector>

#include "oracle.h"

namespace oracle {

// Actions (deprovisioning/types.go): 0 do nothing, 1 delete, 2 replace, 3 retry - a command failed validation.
enum { kActionRetry = 3 };

// A command as Validation reads it: the names of the nodes it removes, 1 delete / 2 replace, and the names of the
// replacement's instance-type options. Commands and the cluster after the TTL meet by name (helpers.go:118-122,328-337).
struct Command {
  std::vector<std::string> nodes;
  int action = 0;
  std::vector<std::string> options;
};

// candidateNodes(after, Validation.ShouldDeprovision) (helpers.go:171-249, validation.go:101-107): Problem.nodes indices in
// node-list order, NOT passed through sortAndFilterCandidates. With derive_candidates off: the nodes marked candidate that
// are not marked for deletion.
std::vector<int> validation_candidates(const kmodel::Problem& after);

// Validation.IsValid + ValidateCommand (validation.go:63-172) against `after`; cands = validation_candidates(after), computed
// once per ComputeCommand (validation.go:78-83, canonical rule R7).
bool is_valid(const kmodel::Problem& after, const std::vector<int>& cands, const Command& cmd);

// The command that removes before.nodes[nodes...] with before.instance_types[options...] as replacement options
Command command_of(const kmodel::Problem& before, const std::vector<int>& nodes, int action, const std::vector<int>& options);

struct ValidatedCommand {
  int action = 0;                 // 0 / 1 / 2 / 3 (retry)
  int position = -1;              // single-node: the winner's position in the disruption order
  int node = -1;                  // single-node: its Problem.nodes index
  int nodes_removed = 0;          // multi-node: prefix of the disruption order the command removes
  std::vector<int> options;
  std::vector<std::pair<int, bool>> validations;  // single-node: (position, valid); multi-node: (nodes_removed, valid)
  bool failed_validation = false;
  ConsolidationResult search;     // multi-node: the search (probes, probe_actions, simulations)
};
// SingleNodeConsolidation.ComputeCommand (singlenodeconsolidation.go:43-84) over positions [first, last) of the disruption
// order (last < 0: all): the first actionable command that validates wins; none, after a failed validation, is retry.
void single_compute_command(const kmodel::Problem& before, const kmodel::Problem& after, int first, int last, ValidatedCommand& out);
// MultiNodeConsolidation.ComputeCommand (multinodeconsolidation.go:41-70): the search, then one validation; invalid -> retry.
void multi_compute_command(const kmodel::Problem& before, const kmodel::Problem& after, ValidatedCommand& out);

}  // namespace oracle
