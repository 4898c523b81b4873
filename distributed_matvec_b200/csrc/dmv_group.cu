// dmv_group.cu -- host-side compilation of a symmetry group into an OrbitProgram.
//
// The reference delegates orbit scans to the third-party ls_hs_state_info / ls_hs_is_representative
// (reference src/FFI.chpl:177-184).  Here the group  G = { t_j . q_i } x {1, flip}  is factored into a
// chain through a subgroup of elements that are cheap as masked shifts (translations) and a right
// transversal applied as Benes networks, so that one orbit scan costs
//     n_q * n_stages butterflies + |G_perm| * (n_left + n_right) masked shifts
// instead of |G_perm| full networks.
#include "dmv_host.h"

#include <algorithm>
#include <map>
#include <random>
#include <set>
#include <stdexcept>

namespace dmv {

namespace {

using Perm = std::vector<int>;  // result bit i = input bit p[i]

Perm compose(const Perm &p, const Perm &q) {  // apply q first, then p:  (p.(q.s))[i] = s[q[p[i]]]
  Perm r(p.size());
  for (size_t i = 0; i < p.size(); ++i) r[i] = q[p[i]];
  return r;
}
Perm inverse(const Perm &p) {
  Perm r(p.size());
  for (size_t i = 0; i < p.size(); ++i) r[p[i]] = (int)i;
  return r;
}
bool is_identity(const Perm &p) {
  for (size_t i = 0; i < p.size(); ++i)
    if (p[i] != (int)i) return false;
  return true;
}

uint64_t apply_naive(const Perm &p, uint64_t s) {
  uint64_t out = 0;
  for (size_t i = 0; i < p.size(); ++i) out |= ((s >> p[i]) & 1ull) << i;
  return out;
}

// masked-shift form: output bit i takes input bit p[i]; d = i - p[i] > 0 is a left shift.
struct ShiftForm {
  std::vector<std::pair<int, uint64_t>> left, right;  // (shift amount, mask over OUTPUT bits)
  int cost() const { return (int)(left.size() + right.size()); }
};
ShiftForm shift_form(const Perm &p) {
  std::map<int, uint64_t> groups;
  for (size_t i = 0; i < p.size(); ++i) groups[(int)i - p[i]] |= 1ull << i;
  ShiftForm f;
  for (auto &kv : groups) {
    if (kv.first >= 0) f.left.push_back({kv.first, kv.second});
    else f.right.push_back({-kv.first, kv.second});
  }
  return f;
}

// Benes routing (looping algorithm).  src[i] = input position that must arrive at output i, width W
// (power of two).  Emits (mask, delta) stages in application order.
void benes_route(std::vector<int> src, int lo_delta_level, int W,
                 std::vector<std::pair<uint64_t, int>> &front,
                 std::vector<std::pair<uint64_t, int>> &back) {
  const int d = W >> (lo_delta_level + 1);
  if (d == 0) return;
  if (d == 1) {
    uint64_t mask = 0;
    for (int p = 0; p < W; p += 2)
      if (src[p] == p + 1) mask |= 1ull << p;
    front.push_back({mask, 1});
    return;
  }
  std::vector<int> dst(W);
  for (int i = 0; i < W; ++i) dst[src[i]] = i;
  std::vector<int> colour_in(W, -1);
  for (int j0 = 0; j0 < W; ++j0) {
    if (colour_in[j0] != -1) continue;
    int j = j0;
    for (;;) {
      colour_in[j] = 0;
      const int jp = j ^ d;          // partner input goes through the upper sub-network
      colour_in[jp] = 1;
      const int ip = dst[jp];        // the output it must reach ...
      const int ipp = ip ^ d;        // ... whose partner output must be fed from the lower sub-network
      const int jn = src[ipp];
      if (colour_in[jn] != -1) break;
      j = jn;
    }
  }
  uint64_t mask_in = 0, mask_out = 0;
  std::vector<int> pos1(W), pos2(W);
  for (int j = 0; j < W; ++j) pos1[j] = colour_in[j] ? (j | d) : (j & ~d);
  for (int i = 0; i < W; ++i) pos2[i] = colour_in[src[i]] ? (i | d) : (i & ~d);
  for (int p = 0; p < W; ++p) {
    if (p & d) continue;
    if (colour_in[p] == 1) mask_in |= 1ull << p;
    if (colour_in[src[p]] == 1) mask_out |= 1ull << p;
  }
  std::vector<int> inner(W);
  for (int i = 0; i < W; ++i) inner[pos2[i]] = pos1[src[i]];
  front.push_back({mask_in, d});
  back.push_back({mask_out, d});
  benes_route(inner, lo_delta_level + 1, W, front, back);
}

std::vector<std::pair<uint64_t, int>> benes_network(const Perm &p, int W) {
  std::vector<int> src(W);
  for (int i = 0; i < W; ++i) src[i] = i;
  for (size_t i = 0; i < p.size(); ++i) src[i] = p[i];
  std::vector<std::pair<uint64_t, int>> front, back;
  benes_route(src, 0, W, front, back);
  std::vector<std::pair<uint64_t, int>> stages = front;
  for (auto it = back.rbegin(); it != back.rend(); ++it) stages.push_back(*it);
  return stages;  // 2 log2(W) - 1 stages, zero masks included
}

struct Candidate {
  std::vector<Perm> chain;      // t_0 = identity, t_1, ...
  std::vector<Perm> steps;      // c_j with t_j = c_j . t_{j-1}
  std::vector<Perm> transversal;
  int n_left = 0, n_right = 0;
  double cost = 0;
};

}  // namespace

HostOrbitProgram compile_orbit_program(int n_sites, int64_t group_order, const int32_t *perms,
                                       const uint8_t *flips, const double *characters) {
  HostOrbitProgram H;
  H.n_sites = n_sites;
  H.site_mask = (n_sites == 64) ? ~0ull : ((1ull << n_sites) - 1);
  if (group_order <= 0) throw std::runtime_error("empty symmetry group");

  // split into permutation part and flip
  std::map<Perm, int> perm_index;
  std::vector<Perm> plist;
  std::map<std::pair<int, int>, std::pair<double, double>> chi;  // (perm idx, flip) -> character
  bool any_flip = false;
  for (int64_t g = 0; g < group_order; ++g) {
    Perm p(perms + g * n_sites, perms + (g + 1) * n_sites);
    auto it = perm_index.find(p);
    int idx;
    if (it == perm_index.end()) {
      idx = (int)plist.size();
      perm_index[p] = idx;
      plist.push_back(p);
    } else idx = it->second;
    const int f = flips[g] ? 1 : 0;
    any_flip |= (f == 1);
    if (chi.count({idx, f})) throw std::runtime_error("duplicate group element");
    chi[{idx, f}] = {characters[2 * g], characters[2 * g + 1]};
  }
  const int Gp = (int)plist.size();
  if ((int64_t)Gp * (any_flip ? 2 : 1) != group_order)
    throw std::runtime_error("group is not a direct product of permutations and spin inversion");
  H.has_flip = any_flip ? 1 : 0;
  bool trivial = true;
  for (auto &kv : chi) trivial &= (kv.second.first == 1.0 && kv.second.second == 0.0);
  H.trivial_characters = trivial ? 1 : 0;

  Perm ident(n_sites);
  for (int i = 0; i < n_sites; ++i) ident[i] = i;
  if (!perm_index.count(ident)) throw std::runtime_error("group lacks the identity");

  const int W = (n_sites > 32) ? 64 : 32;
  const int full_stages = (W == 64) ? 11 : 9;
  std::vector<int> pair_cost(Gp);
  for (int i = 0; i < Gp; ++i) pair_cost[i] = shift_form(plist[i]).cost();

  // candidate factorisations for several "cheap generator" thresholds; kmax = 0: no chain at all
  Candidate best;
  bool have_best = false;
  const double butterfly_cost = (W == 64) ? 8.0 : 4.0, pair_cost_instr = (W == 64) ? 4.0 : 2.0;
  auto build_candidate = [&](const std::vector<Perm> &gens, Candidate &c) -> bool {
    // subgroup generated by gens
    std::set<Perm> T{ident};
    std::vector<Perm> frontier{ident};
    while (!frontier.empty()) {
      std::vector<Perm> nxt;
      for (auto &e : frontier)
        for (auto &g : gens) {
          Perm x = compose(g, e);
          if (T.insert(x).second) nxt.push_back(x);
        }
      frontier.swap(nxt);
    }
    // greedy walk through T
    std::set<Perm> visited{ident};
    c.chain.push_back(ident);
    Perm cur = ident;
    while (visited.size() < T.size()) {
      bool moved = false;
      int best_cost = 1 << 30;
      Perm best_next, best_step;
      for (auto &g : gens) {
        Perm x = compose(g, cur);
        if (!visited.count(x)) {
          const int k = shift_form(g).cost();
          if (k < best_cost) { best_cost = k; best_next = x; best_step = g; moved = true; }
        }
      }
      if (!moved) {  // jump: cheapest connecting element
        const Perm cur_inv = inverse(cur);
        for (auto &x : T) {
          if (visited.count(x)) continue;
          Perm step = compose(x, cur_inv);
          const int k = shift_form(step).cost();
          if (k < best_cost) { best_cost = k; best_next = x; best_step = step; }
        }
      }
      c.chain.push_back(best_next);
      c.steps.push_back(best_step);
      visited.insert(best_next);
      cur = best_next;
    }
    for (auto &s : c.steps) {
      ShiftForm f = shift_form(s);
      c.n_left = std::max(c.n_left, (int)f.left.size());
      c.n_right = std::max(c.n_right, (int)f.right.size());
    }
    // right transversal:  G = union_i T q_i
    std::set<Perm> covered;
    for (auto &p : plist) {
      if (covered.count(p)) continue;
      c.transversal.push_back(p);
      for (auto &t : c.chain) covered.insert(compose(t, p));
    }
    if ((int)covered.size() != Gp || (int)(c.transversal.size() * c.chain.size()) != Gp) return false;
    c.cost = c.transversal.size() * full_stages * butterfly_cost +
             (double)Gp * ((c.n_left + c.n_right) * pair_cost_instr + 8.0);
    return true;
  };
  for (int kmax : {0, 2, 3, 4, 6, 8}) {
    Candidate c;
    std::vector<Perm> gens;
    for (int i = 0; i < Gp; ++i)
      if (!is_identity(plist[i]) && pair_cost[i] <= kmax) gens.push_back(plist[i]);
    if (!build_candidate(gens, c)) continue;
    if (!have_best || c.cost < best.cost) { best = c; have_best = true; }
  }
  if (!have_best) throw std::runtime_error("could not factor the symmetry group");

  // ---- does the group contain the block rotations { rotate the bits inside every k-bit block, rotate the R blocks }
  // (translations of a chain: one block; of an R x k torus numbered row by row)?  Then factor G over THAT subgroup:
  // its orbit minimum needs no walk (translation_canon in dmv_device.cuh), only the coset networks remain.
  if (H.trivial_characters && n_sites >= 2) {
    for (int k = n_sites; k >= 2 && H.canon_mode == 0; --k) {
      if (n_sites % k) continue;
      const int R = n_sites / k;
      if (!(R == 1 || (k <= 8 && R <= 8))) continue;
      Perm A(n_sites), B(n_sites);
      for (int i = 0; i < n_sites; ++i) {
        A[i] = k * (i / k) + ((i % k + 1) % k);   // rotate inside every block
        B[i] = (i + k) % n_sites;                 // rotate the blocks
      }
      if (!perm_index.count(A) || (R > 1 && !perm_index.count(B))) continue;
      Candidate c;
      std::vector<Perm> gens{A};
      if (R > 1) gens.push_back(B);
      if (!build_candidate(gens, c) || (int)c.chain.size() != n_sites) continue;
      best = c;
      H.canon_mode = R == 1 ? 2 : 1;
      H.canon_k = k;
      H.canon_r = R;
    }
  }

  // chains: rotations alone, or rotations x mirror (i -> n-1-i): the whole permutation group in one pass over the runs
  if (H.canon_mode == 2) {
    Perm mirror(n_sites);
    for (int i = 0; i < n_sites; ++i) mirror[i] = n_sites - 1 - i;
    if (best.transversal.size() == 1) H.chain_dihedral = 1;
    else if (best.transversal.size() == 2 && perm_index.count(mirror)) H.chain_dihedral = 2;
  }

  // prefer the identity as the first coset representative (cheaper network: all-zero masks)
  H.n_q = (int)best.transversal.size();
  H.n_t = (int)best.chain.size();
  H.n_left = best.n_left;
  H.n_right = best.n_right;

  // Benes networks of the transversal; keep only stages used by at least one q
  std::vector<std::vector<std::pair<uint64_t, int>>> nets;
  for (auto &q : best.transversal) nets.push_back(benes_network(q, W));
  std::vector<int> keep;
  for (int st = 0; st < full_stages; ++st) {
    bool used = false;
    for (auto &net : nets) used |= (net[st].first != 0);
    if (used) keep.push_back(st);
  }
  H.n_stages = (int)keep.size();
  for (int st : keep) H.benes_delta.push_back(nets[0][st].second);
  for (auto &net : nets)
    for (int st : keep) H.benes_mask.push_back(net[st].first);

  const int n_pairs = H.n_left + H.n_right;
  for (auto &s : best.steps) {
    ShiftForm f = shift_form(s);
    for (int k = 0; k < H.n_left; ++k) {
      if (k < (int)f.left.size()) { H.step_shift.push_back(f.left[k].first); H.step_mask.push_back(f.left[k].second); }
      else { H.step_shift.push_back(0); H.step_mask.push_back(0); }
    }
    for (int k = 0; k < H.n_right; ++k) {
      if (k < (int)f.right.size()) { H.step_shift.push_back(f.right[k].first); H.step_mask.push_back(f.right[k].second); }
      else { H.step_shift.push_back(0); H.step_mask.push_back(0); }
    }
  }
  (void)n_pairs;
  // packed steps for the translation-like fast paths (exactly one left and one right shift per step)
  if (H.n_left == 1 && H.n_right == 1) {
    H.simple = 1;
    for (size_t j = 0; j < best.steps.size(); ++j) {
      const uint64_t ml = H.step_mask[2 * j], mr = H.step_mask[2 * j + 1];
      const uint32_t sl = (uint32_t)H.step_shift[2 * j], sr = (uint32_t)H.step_shift[2 * j + 1];
      H.step_pack64.push_back(ml); H.step_pack64.push_back(mr);
      H.step_pack64.push_back((uint64_t)sl | ((uint64_t)sr << 32));
      if (n_sites <= 32) {
        H.step_pack32.push_back((uint32_t)ml); H.step_pack32.push_back((uint32_t)mr);
        H.step_pack32.push_back(sl); H.step_pack32.push_back(sr);
      }
    }
  }

  if (H.canon_mode == 1) {   // tables of the block-rotation canonical form
    const int k = H.canon_k, R = H.canon_r;
    const uint32_t bm = (1u << k) - 1u;
    H.canon_lut.resize((size_t)1 << k);
    for (uint32_t v = 0; v <= bm; ++v) {
      uint32_t best_v = ~0u, aset = 0;
      for (int a = 0; a < k; ++a) {
        const uint32_t r = a ? (((v >> a) | (v << (k - a))) & bm) : v;
        if (r < best_v) { best_v = r; aset = 1u << a; }
        else if (r == best_v) aset |= 1u << a;
      }
      H.canon_lut[v] = (uint16_t)((aset << 8) | best_v);
    }
    H.canon_masks.assign((size_t)2 * k, 0);
    for (int a = 1; a < k; ++a) {
      uint64_t lo = 0, hi = 0;
      for (int y = 0; y < R; ++y) {
        lo |= (uint64_t)((1u << (k - a)) - 1u) << (k * y);
        hi |= (uint64_t)(bm & ~((1u << (k - a)) - 1u)) << (k * y);
      }
      H.canon_masks[2 * a] = lo;
      H.canon_masks[2 * a + 1] = hi;
    }
  }

  if (H.canon_mode == 1 && 2 * H.canon_k <= 12) {   // pair LUT: top two blocks of a candidate
    const int k = H.canon_k;
    const uint32_t bm = (1u << k) - 1u;
    H.canon_lut2.resize((size_t)1 << (2 * k));
    for (uint32_t hi = 0; hi <= bm; ++hi)
      for (uint32_t lo = 0; lo <= bm; ++lo) {
        uint32_t best_v = ~0u, aset = 0;
        for (int a = 0; a < k; ++a) {
          const uint32_t rh = a ? (((hi >> a) | (hi << (k - a))) & bm) : hi;
          const uint32_t rl = a ? (((lo >> a) | (lo << (k - a))) & bm) : lo;
          const uint32_t v = (rh << k) | rl;
          if (v < best_v) { best_v = v; aset = 1u << a; }
          else if (v == best_v) aset |= 1u << a;
        }
        H.canon_lut2[(hi << k) | lo] = (aset << 16) | best_v;
      }
    H.canon_div = 65536 / k + 1;
    for (int bit = 0; bit < 64; ++bit)
      if (((bit * H.canon_div) >> 16) != bit / k) throw std::runtime_error("canon_div is not exact");
  }
  if (H.canon_mode != 0 && best.transversal.size() > 1) {
    // ---- coset representatives as a chain q_i = c_i . q_{i-1}: c_i a cheap involution of the group (disjoint
    // transpositions grouped by distance = one delta-swap per distinct distance), else a full network
    struct Involution { Perm p; std::map<int, uint64_t> stages; };
    std::vector<Involution> invs;
    for (auto &p : plist) {
      if (is_identity(p) || !is_identity(compose(p, p))) continue;
      Involution v{p, {}};
      for (int i = 0; i < n_sites; ++i)
        if (p[i] > i) v.stages[p[i] - i] |= 1ull << i;
      if (v.stages.size() <= 6) invs.push_back(v);
    }
    std::stable_sort(invs.begin(), invs.end(),
                     [](const Involution &a, const Involution &b) { return a.stages.size() < b.stages.size(); });
    std::map<Perm, int> coset_of;
    for (size_t i = 0; i < best.transversal.size(); ++i)
      for (auto &t : best.chain) coset_of[compose(t, best.transversal[i])] = (int)i;
    std::vector<char> visited(best.transversal.size(), 0);
    Perm cur = ident;
    visited[coset_of.at(ident)] = 1;
    H.cc_begin = {0, 0};   // coset of the identity: no stages
    size_t n_visited = 1;
    while (n_visited < best.transversal.size()) {
      bool moved = false;
      for (auto &v : invs) {
        const Perm x = compose(v.p, cur);
        const int ci = coset_of.at(x);
        if (visited[ci]) continue;
        for (auto &st : v.stages) { H.cc_mask.push_back(st.second); H.cc_delta.push_back(st.first); }
        cur = x; visited[ci] = 1; moved = true;
        break;
      }
      if (!moved) {   // jump to any unvisited coset through a full network
        size_t ci = 0;
        while (visited[ci]) ++ci;
        const Perm step = compose(best.transversal[ci], inverse(cur));
        for (auto &st : benes_network(step, W))
          if (st.first) { H.cc_mask.push_back(st.first); H.cc_delta.push_back(st.second); }
        cur = best.transversal[ci];
        visited[ci] = 1;
      }
      H.cc_begin.push_back((int32_t)H.cc_mask.size());
      ++n_visited;
    }
  }

  // ---- full space group of an R x k torus: block rotations x {1, rho} x {1, sigma} [x {1, tau}]
  // (rho: reverse the bits inside every row, sigma: reverse the order of the rows, tau: transpose).  Then the orbit
  // minimum needs neither the coset chain nor one look-up per (coset, row pair): see orbit_min_torus().
  if (H.canon_mode == 1 && !H.canon_lut2.empty() && H.canon_k >= 3 && H.canon_r >= 3 && 4 * H.canon_r <= 32) {
    const int k = H.canon_k, R = H.canon_r;
    Perm rho(n_sites), sigma(n_sites), tau(n_sites);
    for (int y = 0; y < R; ++y)
      for (int a = 0; a < k; ++a) {
        rho[y * k + a] = y * k + (k - 1 - a);
        sigma[y * k + a] = (R - 1 - y) * k + a;
        tau[y * k + a] = (R == k) ? a * k + y : y * k + a;
      }
    const bool has_tau = R == k && perm_index.count(tau);
    if (perm_index.count(rho) && perm_index.count(sigma)) {
      std::map<Perm, int> coset_of;
      for (size_t i = 0; i < best.transversal.size(); ++i)
        for (auto &t : best.chain) coset_of[compose(t, best.transversal[i])] = (int)i;
      std::vector<Perm> D{ident, rho, sigma, compose(rho, sigma)};
      if (has_tau)
        for (int i = 0; i < 4; ++i) D.push_back(compose(D[i], tau));
      std::set<int> cosets;
      bool ok = true;
      for (auto &d : D) {
        auto it = coset_of.find(d);
        if (it == coset_of.end()) { ok = false; break; }
        cosets.insert(it->second);
      }
      if (ok && cosets.size() == D.size() && D.size() == best.transversal.size()) {
        H.tor_mode = has_tau ? 2 : 1;
        auto add_involution = [&](const Perm &p) {
          std::map<int, uint64_t> stages;
          for (int i = 0; i < n_sites; ++i)
            if (p[i] > i) stages[p[i] - i] |= 1ull << i;
          for (auto &st : stages) { H.tor_net_mask.push_back(st.second); H.tor_net_delta.push_back(st.first); }
          return (int32_t)stages.size();
        };
        H.tor_rho_n = add_involution(rho);
        H.tor_tau_n = has_tau ? add_involution(tau) : 0;
        H.tor_div_r = 65536 / R + 1;
        for (int bit = 0; bit < 32; ++bit)
          if (((bit * H.tor_div_r) >> 16) != bit / R) throw std::runtime_error("tor_div_r is not exact");
        const uint32_t bm = (1u << k) - 1u;
        auto rot = [&](uint32_t v, int a) { return a ? (((v >> a) | (v << (k - a))) & bm) : v; };
        auto rev = [&](uint32_t v) { uint32_t r = 0; for (int b = 0; b < k; ++b) r |= ((v >> b) & 1u) << (k - 1 - b); return r; };
        H.tor_frow.assign((((size_t)4 * k << k) + 15) / 16 * 16, 0);   // padded: staged with 16-byte bulk copies
        for (int f = 0; f < 2; ++f)
          for (int e = 0; e < 2; ++e)
            for (int a = 0; a < k; ++a)
              for (uint32_t r = 0; r <= bm; ++r) {
                uint32_t v = rot(r, a);
                if (e) v = rev(v);
                if (f) v ^= bm;
                H.tor_frow[((size_t)((2 * f + e) * k + a) << k) + r] = (uint8_t)v;
              }
        std::vector<uint16_t> lutm((size_t)1 << (2 * k));
        H.tor_luts.resize((size_t)1 << (2 * k));
        for (uint32_t hi = 0; hi <= bm; ++hi)
          for (uint32_t lo = 0; lo <= bm; ++lo) {
            uint32_t best_v = ~0u, set = 0;
            for (int f = 0; f < (any_flip ? 2 : 1); ++f)
              for (int e = 0; e < 2; ++e)
                for (int a = 0; a < k; ++a) {
                  uint32_t h = rot(hi, a), l = rot(lo, a);
                  if (e) { h = rev(h); l = rev(l); }
                  if (f) { h ^= bm; l ^= bm; }
                  const uint32_t v = (h << k) | l;
                  const uint32_t bit = 1u << ((2 * f + e) * k + a);
                  if (v < best_v) { best_v = v; set = bit; }
                  else if (v == best_v) set |= bit;
                }
            lutm[(hi << k) | lo] = (uint16_t)best_v;
            H.tor_luts[(hi << k) | lo] = set;
          }
        // both orders of a pair in one entry: one look-up per adjacent pair of rows gives the minimum of either order
        H.tor_lutm.resize(lutm.size());
        for (uint32_t hi = 0; hi <= bm; ++hi)
          for (uint32_t lo = 0; lo <= bm; ++lo)
            H.tor_lutm[(hi << k) | lo] = lutm[(hi << k) | lo] | (uint32_t)lutm[(lo << k) | hi] << 16;
      }
    }
  }

  H.characters.resize((size_t)H.n_q * H.n_t * 2 * 2, 0.0);
  for (int q = 0; q < H.n_q; ++q)
    for (int j = 0; j < H.n_t; ++j) {
      const Perm g = compose(best.chain[j], best.transversal[q]);
      const int idx = perm_index.at(g);
      for (int f = 0; f < 2; ++f) {
        std::pair<double, double> c = {1.0, 0.0};
        if (f == 0 || any_flip) c = chi.at({idx, f});
        const size_t e = (((size_t)q * H.n_t + j) * 2 + f) * 2;
        H.characters[e] = c.first;
        H.characters[e + 1] = c.second;
      }
    }
  H.group_order = group_order;

  // self-check against bit-by-bit application on random states
  OrbitProgram P = H.view();
  for (const uint64_t s : orbit_probe_states(H.site_mask)) {
    uint64_t expect = ~0ull;
    int stab = 0;
    for (int i = 0; i < Gp; ++i) {
      const uint64_t y = apply_naive(plist[i], s);
      expect = std::min(expect, y);
      stab += (y == s);
      if (any_flip) { expect = std::min(expect, y ^ H.site_mask); stab += ((y ^ H.site_mask) == s); }
    }
    OrbitResult r = orbit_scan<true, false>(P, s);
    if (r.rep != expect || r.stab != stab) throw std::runtime_error("orbit program self-check failed");
    if (H.canon_mode && orbit_min_canon(P, s) != expect)
      throw std::runtime_error("orbit program self-check failed (canonical form)");
    if (H.tor_mode == 2 && H.canon_k == H.canon_r && (H.canon_k == 4 || H.canon_k == 6)) {
      const uint64_t got = H.canon_k == 6 ? orbit_min_torus_sq<6>(P, s) : orbit_min_torus_sq<4>(P, s);
      if (got != expect) throw std::runtime_error("orbit program self-check failed (square-torus form)");
    }
    if (H.tor_mode || H.chain_dihedral) {   // the forms underneath stay selectable (option "canon" = 1): check them as well
      OrbitProgram P1 = P;
      P1.tor_mode = 0;
      P1.chain_dihedral = 0;
      if (orbit_min_canon(P1, s) != expect)
        throw std::runtime_error("orbit program self-check failed (block-rotation canonical form)");
    }
    // the element reported as minimising must really map s to rep
    const int e = r.arg >> 1;
    const Perm g = compose(best.chain[e % H.n_t], best.transversal[e / H.n_t]);
    uint64_t y = apply_naive(g, s);
    if (r.arg & 1) y ^= H.site_mask;
    if (y != r.rep) throw std::runtime_error("orbit program argmin self-check failed");
  }
  return H;
}

std::vector<uint64_t> orbit_probe_states(uint64_t site_mask) {
  std::mt19937_64 rng(12345);
  // random states plus patterns with many tied rotations (uniform, alternating, repeated blocks, single bits)
  std::vector<uint64_t> probes = {0ull, site_mask, 0x5555555555555555ull & site_mask,
                                  0xaaaaaaaaaaaaaaaaull & site_mask, 1ull, site_mask >> 1,
                                  0x3333333333333333ull & site_mask, 0x0f0f0f0f0f0f0f0full & site_mask,
                                  0x249249249249249ull & site_mask, 0x1041041041041041ull & site_mask};
  for (int trial = 0; trial < 256; ++trial) {
    uint64_t v = rng() & site_mask;
    if (trial & 1) v &= rng();            // sparse and dense words: long runs
    if ((trial & 3) == 3) v = ~v & site_mask;
    probes.push_back(v);
  }
  return probes;
}

namespace {
template <int K>
bool torus_sq_rows_check_k(const OrbitProgram &P, const std::vector<uint64_t> &flips) {
  for (const uint64_t s : orbit_probe_states(P.site_mask)) {
    const uint64_t st = torus_sq_columns<K>(s);
    for (const uint64_t x : flips) {
      const uint64_t w = (s ^ x) & P.site_mask;
      if (orbit_min_torus_sq_t<K>(P, w, st ^ torus_sq_columns<K>(x & P.site_mask)) != orbit_min_torus_sq<K>(P, w))
        return false;
    }
  }
  return true;
}
}  // namespace

bool torus_sq_rows_check(const OrbitProgram &P, const std::vector<uint64_t> &flips) {
  if (P.canon_k == 6) return torus_sq_rows_check_k<6>(P, flips);
  if (P.canon_k == 4) return torus_sq_rows_check_k<4>(P, flips);
  return false;
}

OrbitProgram HostOrbitProgram::view() const {
  OrbitProgram P;
  P.n_sites = n_sites;
  P.n_q = n_q; P.n_stages = n_stages; P.n_t = n_t; P.n_left = n_left; P.n_right = n_right;
  P.has_flip = has_flip; P.trivial_characters = trivial_characters;
  P.site_mask = site_mask;
  P.benes_mask = benes_mask.data();
  P.benes_delta = benes_delta.data();
  P.step_mask = step_mask.data();
  P.step_shift = step_shift.data();
  P.characters = reinterpret_cast<const double2 *>(characters.data());
  P.group_order = group_order;
  P.simple = simple;
  P.step_pack32 = step_pack32.empty() ? nullptr : reinterpret_cast<const uint4 *>(step_pack32.data());
  P.step_pack64 = step_pack64.data();
  P.canon_mode = canon_mode; P.canon_k = canon_k; P.canon_r = canon_r;
  P.chain_dihedral = chain_dihedral;
  P.canon_lut = canon_lut.data();
  P.canon_masks = canon_masks.data();
  P.canon_lut2 = canon_lut2.empty() ? nullptr : canon_lut2.data();
  P.canon_div = canon_div;
  P.cc_n = cc_begin.empty() ? 0 : (int32_t)cc_begin.size() - 1;
  P.cc_stages = (int32_t)cc_mask.size();
  P.cc_begin = cc_begin.data();
  P.cc_mask = cc_mask.data();
  P.cc_delta = cc_delta.data();
  P.tor_mode = tor_mode; P.tor_rho_n = tor_rho_n; P.tor_tau_n = tor_tau_n; P.tor_div_r = tor_div_r;
  P.tor_sq_rows = 0;
  P.tor_lutm = tor_lutm.data();
  P.tor_luts = tor_luts.data();
  P.tor_frow = tor_frow.data();
  P.tor_net_mask = tor_net_mask.data();
  P.tor_net_delta = tor_net_delta.data();
  return P;
}

}  // namespace dmv
