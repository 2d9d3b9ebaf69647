// teaser::Graph / teaser::MaxCliqueSolver — the public graph façade of the reference
// (teaser/include/teaser/graph.h:29-279), kept source compatible.  Graph is the same adjacency-list
// container; MaxCliqueSolver::findMaxClique forwards to the GPU C-ABI (tzr_max_clique) instead of PMC.
#pragma once
#include <algorithm>
#include <map>
#include <vector>

namespace teaser {

class Graph {
 public:
  Graph() = default;
  explicit Graph(const std::map<int, std::vector<int>>& adj_list) {
    adj_.resize(adj_list.size());
    size_t twice = 0;
    for (const auto& kv : adj_list) {
      adj_[kv.first] = kv.second;
      twice += kv.second.size();
    }
    num_edges_ = twice / 2;
  }
  void addVertex(const int& id) {
    if (id >= static_cast<int>(adj_.size())) adj_.resize(id + 1);
  }
  void populateVertices(const int& n) { adj_.resize(n); }
  bool hasEdge(const int& a, const int& b) const {
    if (a >= static_cast<int>(adj_.size()) || b >= static_cast<int>(adj_.size())) return false;
    return std::find(adj_[a].begin(), adj_[a].end(), b) != adj_[a].end();
  }
  bool hasVertex(const int& v) const { return v < static_cast<int>(adj_.size()); }
  void addEdge(const int& a, const int& b) {
    if (hasEdge(a, b)) return;
    adj_[a].push_back(b);
    adj_[b].push_back(a);
    ++num_edges_;
  }
  void removeEdge(const int& a, const int& b) {
    if (a >= static_cast<int>(adj_.size()) || b >= static_cast<int>(adj_.size())) return;
    auto drop = [](std::vector<int>& v, int x) { v.erase(std::remove(v.begin(), v.end(), x), v.end()); };
    drop(adj_[a], b);
    drop(adj_[b], a);
    --num_edges_;
  }
  int numVertices() const { return static_cast<int>(adj_.size()); }
  int numEdges() const { return static_cast<int>(num_edges_); }
  const std::vector<int>& getEdges(int id) const { return adj_[id]; }
  std::vector<int> getVertices() const {
    std::vector<int> v(adj_.size());
    for (size_t i = 0; i < v.size(); ++i) v[i] = static_cast<int>(i);
    return v;
  }
  std::vector<std::vector<int>> getAdjList() const { return adj_; }
  void setAdjList(std::vector<std::vector<int>> adj, size_t edges) {
    adj_ = std::move(adj);
    num_edges_ = edges;
  }
  void reserve(const int& n) { adj_.reserve(n); }
  void clear() {
    adj_.clear();
    num_edges_ = 0;
  }

 private:
  std::vector<std::vector<int>> adj_;
  size_t num_edges_ = 0;
};

class MaxCliqueSolver {
 public:
  enum class CLIQUE_SOLVER_MODE { PMC_EXACT = 0, PMC_HEU = 1, KCORE_HEU = 2 };
  struct Params {
    CLIQUE_SOLVER_MODE solver_mode = CLIQUE_SOLVER_MODE::PMC_EXACT;
    bool solve_exactly = true;  // deprecated in the reference
    double kcore_heuristic_threshold = 1;
    double time_limit = 3600;
    int num_threads = 1;  // ignored on the GPU
  };
  MaxCliqueSolver() = default;
  explicit MaxCliqueSolver(Params params) : params_(params) {}
  // teaser/src/graph.cc:12-125 — returns the clique sorted ascending
  std::vector<int> findMaxClique(Graph graph);

 private:
  Params params_;
};

}  // namespace teaser
