// kp_slot.hpp -- the node-selector set algebra of pkg/scheduling/requirement.go on one 64-bit value mask per key.
// Host + device. A Slot is one scheduling.Requirement: {complement, values (mask over the key's interned values), gte, lte}.
// An absent slot (flags without SF_PRESENT) reads as "Exists" where the reference's Requirements.Get does
// (requirements.go:160-166).
#pragma once
#include <cstdint>

#include "kp_tables.hpp"

#ifdef __CUDACC__
#define KP_HD __host__ __device__ __forceinline__
#else
#define KP_HD inline
#endif


struct KeyInfo {  // integer reading of a key's values (strconv.Atoi, requirement.go:326-342)
  const int64_t* val_int;  // [64]
  uint64_t isint;
  uint64_t univ;
};

KP_HD Slot slot_absent() { return Slot{0u, 0ull, 0, 0}; }
KP_HD Slot slot_exists() { return Slot{SF_PRESENT | SF_COMPLEMENT, 0ull, 0, 0}; }
KP_HD bool slot_present(const Slot& s) { return s.f & SF_PRESENT; }

KP_HD bool slot_eq(const Slot& a, const Slot& b) {
  if (a.f != b.f || a.m != b.m) return false;
  if ((a.f & SF_HAS_GTE) && a.gte != b.gte) return false;
  if ((a.f & SF_HAS_LTE) && a.lte != b.lte) return false;
  return true;
}

// requirement.go:282-293 Operator()
KP_HD int slot_op(const Slot& s) {
  if (s.f & SF_COMPLEMENT) return s.m ? OP_NOT_IN : OP_EXISTS;
  return s.m ? OP_IN : OP_DNE;
}
KP_HD bool op_is_negative(int op) { return op == OP_NOT_IN || op == OP_DNE; }

// values of the key's universe that satisfy the bounds (withinBounds, requirement.go:326-342)
KP_HD uint64_t bounds_mask(const KeyInfo& ki, bool hg, int64_t g, bool hl, int64_t l) {
  if (!hg && !hl) return ~0ull;
  uint64_t out = 0;
  uint64_t cand = ki.isint;
  while (cand) {
#ifdef __CUDA_ARCH__
    int v = __ffsll((long long)cand) - 1;
#else
    int v = __builtin_ctzll(cand);
#endif
    cand &= cand - 1;
    int64_t x = ki.val_int[v];
    if (hg && x < g) continue;
    if (hl && x > l) continue;
    out |= 1ull << v;
  }
  return out;
}

KP_HD void combine_bounds(const Slot& a, const Slot& b, bool* hg, int64_t* g, bool* hl, int64_t* l) {
  bool ag = a.f & SF_HAS_GTE, bg = b.f & SF_HAS_GTE, al = a.f & SF_HAS_LTE, bl = b.f & SF_HAS_LTE;
  *hg = ag || bg;
  *g = (ag && bg) ? (a.gte > b.gte ? a.gte : b.gte) : (ag ? a.gte : b.gte);
  *hl = al || bl;
  *l = (al && bl) ? (a.lte < b.lte ? a.lte : b.lte) : (al ? a.lte : b.lte);
}

// requirement.go:212-246 HasIntersection (both slots present)
KP_HD bool slot_has_intersection(const KeyInfo& ki, const Slot& a, const Slot& b) {
  bool hg, hl;
  int64_t g, l;
  combine_bounds(a, b, &hg, &g, &hl, &l);
  if (hg && hl && g > l) return false;
  bool ac = a.f & SF_COMPLEMENT, bc = b.f & SF_COMPLEMENT;
  if (ac && bc) return true;
  uint64_t inb = bounds_mask(ki, hg, g, hl, l);
  if (ac) return (b.m & ~a.m & inb) != 0;
  if (bc) return (a.m & ~b.m & inb) != 0;
  return (a.m & b.m & inb) != 0;
}

// requirement.go:173-206 Intersection (both slots present)
KP_HD Slot slot_intersection(const KeyInfo& ki, const Slot& a, const Slot& b) {
  bool hg, hl;
  int64_t g, l;
  combine_bounds(a, b, &hg, &g, &hl, &l);
  Slot o;
  o.gte = 0;
  o.lte = 0;
  if (hg && hl && g > l) {  // DoesNotExist
    o.f = SF_PRESENT;
    o.m = 0;
    return o;
  }
  bool ac = a.f & SF_COMPLEMENT, bc = b.f & SF_COMPLEMENT;
  uint64_t vals;
  if (ac && bc)
    vals = a.m | b.m;
  else if (ac)
    vals = b.m & ~a.m;
  else if (bc)
    vals = a.m & ~b.m;
  else
    vals = a.m & b.m;
  vals &= bounds_mask(ki, hg, g, hl, l);
  o.m = vals;
  o.f = SF_PRESENT;
  if (ac && bc) {
    o.f |= SF_COMPLEMENT;
    if (hg) {
      o.f |= SF_HAS_GTE;
      o.gte = g;
    }
    if (hl) {
      o.f |= SF_HAS_LTE;
      o.lte = l;
    }
  }
  return o;
}

// Requirements.Add (requirements.go:133-140): incoming.Intersection(existing), or insert
KP_HD Slot slot_add(const KeyInfo& ki, const Slot& existing, const Slot& incoming) {
  if (!slot_present(incoming)) return existing;
  if (!slot_present(existing)) return incoming;
  return slot_intersection(ki, incoming, existing);
}

// requirement.go:267-272 Has(value); absent slot == Exists
KP_HD bool slot_has(const KeyInfo& ki, const Slot& s, int v) {
  if (!slot_present(s)) return true;
  bool in = (s.m >> v) & 1;
  bool hg = s.f & SF_HAS_GTE, hl = s.f & SF_HAS_LTE;
  bool wb = true;
  if (hg || hl) {
    wb = (ki.isint >> v) & 1;
    if (wb) {
      int64_t x = ki.val_int[v];
      if (hg && x < s.gte) wb = false;
      if (hl && x > s.lte) wb = false;
    }
  }
  return ((s.f & SF_COMPLEMENT) ? !in : in) && wb;
}
// mask of universe values the slot allows (Has(v) for every v)
KP_HD uint64_t slot_allowed(const KeyInfo& ki, const Slot& s) {
  if (!slot_present(s)) return ki.univ;
  uint64_t inb = bounds_mask(ki, s.f & SF_HAS_GTE, s.gte, s.f & SF_HAS_LTE, s.lte);
  return ((s.f & SF_COMPLEMENT) ? ~s.m : s.m) & inb & ki.univ;
}

// One key of Requirements.Compatible(existing <- incoming) (requirements.go:181-197,254-274).
// Returns true when this key raises no error.
KP_HD bool slot_compatible(const KeyInfo& ki, const Slot& existing, const Slot& incoming, bool well_known,
                           bool allow_undefined) {
  if (!slot_present(incoming)) return true;
  if (!slot_present(existing)) {
    if (allow_undefined && well_known) return true;            // Intersects skips keys that are not shared
    return op_is_negative(slot_op(incoming));                  // "label does not have known values"
  }
  if (slot_has_intersection(ki, existing, incoming)) return true;
  return op_is_negative(slot_op(incoming)) && op_is_negative(slot_op(existing));
}
// ---- the same algebra when no requirement in the problem carries Gt / Lt bounds (has_bounds == 0): flags + mask only
KP_HD bool slot_neg_nb(const Slot& s) { return ((s.f & SF_COMPLEMENT) != 0) == (s.m != 0); }  // NotIn or DoesNotExist
KP_HD bool slot_compatible_nb(const Slot& existing, const Slot& incoming, bool well_known, bool allow_undefined) {
  if (!(incoming.f & SF_PRESENT)) return true;
  if (!(existing.f & SF_PRESENT)) return (allow_undefined && well_known) || slot_neg_nb(incoming);
  const bool ac = existing.f & SF_COMPLEMENT, bc = incoming.f & SF_COMPLEMENT;
  bool inter;
  if (ac && bc)
    inter = true;
  else if (ac)
    inter = (incoming.m & ~existing.m) != 0;
  else if (bc)
    inter = (existing.m & ~incoming.m) != 0;
  else
    inter = (existing.m & incoming.m) != 0;
  return inter || (slot_neg_nb(incoming) && slot_neg_nb(existing));
}
KP_HD Slot slot_add_nb(const Slot& existing, const Slot& incoming) {
  if (!(incoming.f & SF_PRESENT)) return existing;
  if (!(existing.f & SF_PRESENT)) return incoming;
  const bool ac = incoming.f & SF_COMPLEMENT, bc = existing.f & SF_COMPLEMENT;
  Slot o;
  o.gte = 0;
  o.lte = 0;
  o.f = SF_PRESENT | ((ac && bc) ? SF_COMPLEMENT : 0u);
  if (ac && bc)
    o.m = incoming.m | existing.m;
  else if (ac)
    o.m = existing.m & ~incoming.m;
  else if (bc)
    o.m = incoming.m & ~existing.m;
  else
    o.m = incoming.m & existing.m;
  return o;
}

// The host rule of requirement set rs (KpDev::host_rules) on hostname domain `host`: an existing node (host < E) is
// admitted iff its hostname satisfies the rule, a NodeClaim iff the rule is a complement (NotIn / Exists).  Every
// NodeClaim carries hostname In{placeholder} that no pod can name (nodeclaim.go:92-96), every existing node hostname
// In{its hostname} (existingnode.go:62), so a rule never changes a candidate's requirements, only admits or rejects it.
KP_HD bool host_rule_admits(const int32_t* host_rules, int E, int rs, int host) {
  const int o = host_rules[rs];
  if (o < 0) return true;
  return host < E ? (((uint32_t)host_rules[o + 1 + (host >> 5)] >> (host & 31)) & 1u) != 0 : host_rules[o] != 0;
}
