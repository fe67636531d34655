// schema.h -- SpiceDB schema DSL subset -> flat device program.
//
// The reference configures its engine with schema text (pkg/spicedb/bootstrap.yaml:1-38,
// pkg/spicedb/spicedb.go:19-24). This compiler turns that text into the tables the
// CUDA kernels walk:
//   * every relation becomes a "data relation" with one EDGE CLASS per allowed
//     subject kind (type, type#rel, type:*): subject type and child slot are static
//     per class, so an edge is a bare u32 object id;
//   * every permission whose (same-object-inlined) expression is a pure union
//     becomes a UNIT: a short list of REL / ARROW ops evaluated as reachability;
//   * permissions containing & or - become a TREE: a postfix boolean program over
//     leaf units, evaluated after the reachability pass (DESIGN.md "Boolean
//     structure").
#pragma once
#include <cstdint>
#include <string>
#include <vector>

namespace zg {

constexpr uint16_t kNone = 0xFFFF;      // ZG_SREL_NONE
constexpr uint16_t kWildcard = 0xFFFE;  // ZG_SREL_WILDCARD
constexpr int kMaxClasses = 8;          // edge classes per relation
constexpr int kMaxLeaves = 32;          // leaf units per non-pure permission

// ---- device-visible PODs (copied verbatim into the program blob) -------------
enum SlotKind : uint16_t { SK_RELATION = 0, SK_PURE = 1, SK_NONPURE = 2 };
enum OpKind : uint16_t { OP_REL = 0, OP_ARROW = 1 };
enum TreeOpKind : uint16_t { T_LEAF = 0, T_TRIVIAL = 1, T_OR = 2, T_AND = 3, T_ANDNOT = 4 };
enum ClsFlags : uint16_t {
  CF_EXPIRY = 1,  // relationships of this class may carry an expiration
  CF_EMPTY = 2,   // no relationship of this class in the whole snapshot (set at publish)
  CF_INVERT = 4,  // direct class whose probes may be answered from the subject's reverse row
};
enum UnitFlags : uint16_t {
  UF_EXPANSIVE = 1,  // unit can push userset / arrow ranges
  UF_LEAF_INV = 2,   // in this snapshot every step is an invertible direct probe: a visit can
                     // only answer "is (class, obj) one of the subject's own memberships"
};
constexpr uint16_t kStepTargetLeaf = 0x100;  // DStep.flags: children are UF_LEAF_INV visits
constexpr uint16_t kStepTargetL2 = 0x200;    // DStep.flags: the children's unit is ONE userset edge class whose own
                                             // children are UF_LEAF_INV visits (resource -> team#member -> user): the
                                             // whole two-level range is answered from the subject's reverse rows

enum SlotFlags : uint16_t {
  SF_NO_RSET = 1,  // no step of a unit the slot evaluates at the root reads the subject's per-check membership set
                   // (set at publish once the closure indexes are built: mark_rsetless_slots)
  SF_FLAT = 2,     // the slot's checks are answered by flat_check_kernel (kernels.cuh): SF_NO_RSET, a pure slot whose
                   // push steps (1 .. kFlatSteps) all meet over closure indexes with signatures and set tables
                   // (mark_flat_slots)
};
constexpr int kFlatSteps = 4;       // push steps of an SF_FLAT slot, at most
constexpr int kMaxInvClasses = 11;  // invertible classes of a subject type the check kernel's admission takes
struct DSlot {   // per slot (relation or permission)
  uint16_t kind;        // SlotKind
  uint16_t unit;        // SK_RELATION / SK_PURE: unit id ; SK_NONPURE: tree id
  uint16_t type;
  uint16_t flags;       // SlotFlags
};
struct DUnit {   // pure-union program evaluated at one object
  uint16_t op_begin, op_end;    // into ops[]
  uint16_t mem_begin, mem_end;  // into members[]: slots inlined into this unit
  uint16_t flags;               // UnitFlags
  uint16_t step_begin, step_end;  // into steps[]: the unit flattened for this snapshot, probes first:
  uint16_t push_begin;            // [step_begin, push_begin) DIRECT / WILD (lane-local), [push_begin, step_end) PUSH
};
// One edge class a unit touches, with everything the visit needs in one 24-byte record.
// Built at publish: classes that are empty in the snapshot produce no step at all.
enum StepKind : uint16_t { ST_DIRECT = 0, ST_WILD = 1, ST_PUSH = 2 };
struct DStep {
  uint64_t row_base;  // row_ptr index of (object 0, this class): rel.row_base + k
  uint32_t nres;      // objects covered by the relation's row table
  uint16_t ncls;      // row stride per object (all classes of the resource type)
  uint16_t kind;      // StepKind
  uint16_t stype;     // ST_DIRECT / ST_WILD: subject type that can match
  uint16_t tslot;     // ST_PUSH: slot the children are visited at
  uint16_t flags;     // ClsFlags (CF_EXPIRY, CF_INVERT) | kStepTargetLeaf
  uint16_t gc;        // global class id (key of the subject's reverse-row set)
  uint16_t tunit;     // ST_PUSH: unit of tslot (kNone when tslot is a non-pure permission)
  uint16_t tgc;       // kStepTargetLeaf: the single class of the target unit; kStepTargetL2: the single
                      // (userset) class of the target unit, whose reverse rows are streamed
  uint16_t tinv;      // ST_DIRECT: index of gc among its subject type's invertible classes;
                      // kStepTargetLeaf: the same for tgc; kStepTargetL2: for the innermost direct class
  uint16_t tstype;    // kStepTargetLeaf / kStepTargetL2: subject type the (innermost) direct class accepts
};
struct DOp {
  uint16_t kind;       // OpKind
  uint16_t rel;        // data relation index
  uint16_t tgt_begin;  // OP_ARROW: tgts[tgt_begin + class] = child slot or kNone
  uint16_t pad;
};
struct DRel {    // data relation: rows of (object x class). All relations of one resource type
                 // are interleaved per object, so one object's offsets share a sector or two.
  uint64_t row_base;   // index into row_ptr pool of (object 0, class 0 of this relation)
  uint32_t nres;       // objects covered
  uint16_t ncls;       // classes of this relation
  uint16_t cls_begin;  // into classes[]
  uint32_t stride;     // classes of ALL relations of the resource type = row stride per object
  uint32_t pad;
};
struct DCls {
  uint16_t stype;
  uint16_t sslot;      // kNone (direct), kWildcard, or subject relation slot
  uint16_t flags;      // ClsFlags
  uint16_t rel;        // data relation index this class belongs to
  uint32_t nsubj;      // reverse CSR: subject objects covered (1 for a wildcard class)
  uint16_t rtype;      // type of the resources of this class
  uint16_t rstride;    // reverse CSR row stride per subject: the reverse rows of ALL classes of one
                       // subject type are interleaved per subject (one or two sectors hold every
                       // offset of a subject), like the forward tables are per object
  uint64_t rrow_base;  // reverse CSR: rrow_ptr index of (subject 0, this class); row of subject s =
                       // rrow_base + s * rstride
};
struct FwdClass {  // LookupSubjects' forward walk: one non-wildcard edge class, grouped by resource type
  uint64_t row_base;  // row_ptr index of (object 0, this class)
  uint32_t nres;      // objects covered by the relation's row table
  uint16_t ncls;      // row stride per object
  uint16_t stype;     // type of the subjects (the children)
  uint16_t gc;        // global class id (bit of Schema::fwd_mask)
  uint16_t pad[3];
};
struct DTypeInv {  // per subject type: the invertible direct classes (inv_cls[begin, end))
  uint16_t begin, end;
};
// ExpandPermissionTree (expand.cuh): every slot lowered into a pre-order template of the tree one object contributes.
// Same-object references are inlined; arrows end the template, their children are the next level's jobs.
enum XOpKind : uint16_t { X_UNION = 1, X_INTER = 2, X_EXCL = 3, X_REL = 4, X_NIL = 5, X_ARROW = 6 };
constexpr int kMaxExpandTemplate = 32;  // nodes of one template: a warp writes them, one per lane
struct XNode {
  uint16_t op;      // XOpKind
  uint16_t slot;    // the expanded relation
  uint8_t parent;   // template index of the parent (0 at the root, which has none)
  uint8_t rank;     // position among the parent's children
  uint8_t count;    // X_REL / X_ARROW: index among the template's counted nodes
  uint8_t size;     // root only: nodes of the template
  uint8_t ncount;   // root only: counted (X_REL / X_ARROW) nodes
  uint8_t pad;
  uint16_t rel;     // X_REL: data relation; X_ARROW: the tupleset's data relation
  uint32_t tgt;     // X_ARROW: x_tgts[tgt + k] = template root of class k's target, kNoTemplate: an empty leaf
  uint32_t counted; // root only: x_counted[counted + i] = template index of counted node i
};
constexpr uint32_t kNoTemplate = 0xFFFFFFFFu;

struct DTree {   // postfix boolean program of a non-pure permission
  uint16_t op_begin, op_end;     // into tree_ops[]
  uint16_t leaf_begin, n_leaves; // leaf_units[leaf_begin + i] = unit id
  uint16_t flags;                // UF_EXPANSIVE when any leaf unit is
  uint16_t pad;
};
struct DTreeOp {
  uint16_t kind;  // TreeOpKind
  uint16_t arg;   // T_LEAF: leaf index ; T_TRIVIAL: slot
};
struct DHeader {  // first bytes of the blob; offsets in bytes from blob start
  uint32_t magic, total_bytes;
  uint32_t n_types, n_slots, n_units, n_ops, n_rels, n_cls, n_trees, n_tree_ops;
  uint32_t off_slots, off_units, off_ops, off_rels, off_cls, off_tgts, off_members;
  uint32_t off_trees, off_tree_ops, off_leaf_units, off_reach;
  uint32_t off_type_inv, off_inv_cls, off_steps, n_steps;
  uint32_t off_type_rcls, off_rcls;  // per subject type: every class whose subjects have that type
  uint32_t max_leaves;   // job stride L in general mode (1 if no non-pure slot)
  uint32_t has_nonpure;
  uint32_t has_expiry;
  uint32_t reach_words;  // u32 words per slot in reach[] (bit t: subjects of type t reachable)
};

// ---- host-side model -----------------------------------------------------------
struct ClassInfo {
  uint16_t stype;
  uint16_t sslot;
  bool expiry;
};
struct Expr {
  enum Kind { NIL, REF, ARROW, UNION, INTER, EXCL } kind = NIL;
  int slot = -1;   // REF: slot ; ARROW: tupleset relation slot
  int name = -1;   // ARROW: name id of the computed permission
  int l = -1, r = -1;
};
struct SlotInfo {
  std::string name;
  int name_id = -1;
  uint16_t type = 0;
  bool is_perm = false;
  std::vector<ClassInfo> classes;  // relations
  int expr = -1;                   // permissions: root in Schema::exprs
  int rel_index = -1;              // relations: data relation index
  uint16_t kind = SK_RELATION;
  int unit = -1, tree = -1;
};
struct TypeInfo {
  std::string name;
  std::vector<int> slots;
};

class Schema {
 public:
  // Returns empty string on success, else the error message.
  std::string parse(const std::string& text);

  int type_id(const std::string& n) const;
  int slot_id(int type, const std::string& n) const;
  int slot_by_name_id(int type, int name_id) const;
  int class_of(int rel_slot, uint16_t stype, uint16_t sslot) const;  // -1 if not allowed

  std::vector<TypeInfo> types;
  std::vector<SlotInfo> slots;
  std::vector<std::string> names;
  std::vector<Expr> exprs;
  std::vector<int> rel_slots;  // data relation index -> slot
  bool use_expiration = false;

  // compiled tables
  std::vector<DSlot> d_slots;
  std::vector<DUnit> d_units;
  std::vector<DOp> d_ops;
  std::vector<DCls> d_cls;
  std::vector<uint16_t> d_tgts, d_members, d_leaf_units;
  std::vector<DTree> d_trees;
  std::vector<DTreeOp> d_tree_ops;
  std::vector<uint32_t> d_reach;
  uint32_t reach_words = 1;
  uint32_t max_leaves = 1;
  bool has_nonpure = false, has_expiry = false;

  // Serialises the program; DRel rows (row_base, nres) come from the store.
  // cls: per-class dynamic data from the store (rrow_base, CF_EMPTY), same order as d_cls.
  std::vector<uint8_t> blob(const std::vector<DRel>& rels, const std::vector<DCls>& cls) const;
  std::vector<DTypeInv> d_type_inv, d_type_rcls;
  std::vector<uint16_t> d_inv_cls, d_rcls;
  // LookupSubjects: per slot, fwd_mask_words words whose bit gc says that class gc is read by the slot's
  // evaluation (the closure over REL / ARROW ops and userset child slots, wildcard classes excluded).
  std::vector<uint32_t> fwd_mask;
  uint32_t fwd_mask_words = 1;
  // Per resource type, its relations' non-wildcard classes with their rows in this snapshot's layout:
  // fwd[type_off[t], type_off[t + 1]).
  void forward_tables(const std::vector<DRel>& rels, std::vector<FwdClass>* fwd, std::vector<uint32_t>* type_off) const;
  // ExpandPermissionTree templates (XNode): x_root[slot] = root of the slot's template in x_nodes. x_ok[slot] = 0 when
  // its template, or one an arrow of it reaches, has more than kMaxExpandTemplate nodes: expanding it is refused.
  std::vector<XNode> x_nodes;
  std::vector<uint32_t> x_tgts, x_counted, x_root;
  std::vector<uint8_t> x_ok;

 private:
  void compute_forward_masks();
  void compute_expand_templates();
  std::string compile();
  int name_id(const std::string& n);
};

// Sets SF_NO_RSET in the slot table of a program blob (Schema::blob) for every slot whose checks never read the
// per-check membership set: in every unit the slot evaluates at the root, no probe step is an invertible direct
// class (CF_INVERT) and every push step is a two-level step (kStepTargetL2) whose class has a closure index
// (indexed_tgc lists the tgc of every pair built). Returns the number of slots marked.
int mark_rsetless_slots(std::vector<uint8_t>* blob, const std::vector<uint16_t>& indexed_tgc);

// Sets SF_FLAT (and clears it elsewhere) in a program blob whose SF_NO_RSET flags are marked, for every pure slot that
// has SF_NO_RSET, between 1 and kFlatSteps push steps, every one of them over a pair in tabled_tgc (the tgc of every
// pair built with signatures and set tables), and whose two-level steps' subject types have at most kMaxInvClasses
// invertible classes. Pass an empty tabled_tgc to clear every flag. Returns the number of slots marked.
int mark_flat_slots(std::vector<uint8_t>* blob, const std::vector<uint16_t>& tabled_tgc);

}  // namespace zg
