// schema.cc -- parser + compiler for the SpiceDB schema DSL subset used by the
// reference (pkg/spicedb/bootstrap.yaml:1-38, e2e/embedded_integration_test.go:56-93,
// pkg/proxy/options_test.go:226-237). See schema.h for the output model.
#include "schema.h"

#include <algorithm>
#include <cctype>
#include <cstring>
#include <functional>
#include <stdexcept>

namespace zg {

namespace {

struct Token {
  enum Kind { END, IDENT, SYM } kind = END;
  std::string text;
  int line = 1;
};

class Scanner {
 public:
  explicit Scanner(const std::string& s) : s_(s) { advance(); }
  const Token& peek() const { return cur_; }
  Token take() {
    Token t = cur_;
    advance();
    return t;
  }
  bool is_sym(const char* sym) const { return cur_.kind == Token::SYM && cur_.text == sym; }
  bool is_word(const char* w) const { return cur_.kind == Token::IDENT && cur_.text == w; }
  [[noreturn]] void fail(const std::string& msg) const {
    throw std::runtime_error("schema line " + std::to_string(cur_.line) + ": " + msg +
                             (cur_.kind == Token::END ? " (at end of input)" : " (near '" + cur_.text + "')"));
  }
  void expect_sym(const char* sym) {
    if (!is_sym(sym)) fail(std::string("expected '") + sym + "'");
    advance();
  }
  std::string expect_ident(const char* what) {
    if (cur_.kind != Token::IDENT) fail(std::string("expected ") + what);
    return take().text;
  }

 private:
  void advance() {
    for (;;) {
      while (i_ < s_.size() && std::isspace(static_cast<unsigned char>(s_[i_]))) {
        if (s_[i_] == '\n') ++line_;
        ++i_;
      }
      if (i_ + 1 < s_.size() && s_[i_] == '/' && s_[i_ + 1] == '/') {
        while (i_ < s_.size() && s_[i_] != '\n') ++i_;
        continue;
      }
      if (i_ + 1 < s_.size() && s_[i_] == '/' && s_[i_ + 1] == '*') {
        i_ += 2;
        while (i_ + 1 < s_.size() && !(s_[i_] == '*' && s_[i_ + 1] == '/')) {
          if (s_[i_] == '\n') ++line_;
          ++i_;
        }
        i_ = std::min(i_ + 2, s_.size());
        continue;
      }
      break;
    }
    cur_ = Token{};
    cur_.line = line_;
    if (i_ >= s_.size()) return;
    unsigned char c = static_cast<unsigned char>(s_[i_]);
    if (std::isalpha(c) || c == '_') {
      size_t b = i_;
      while (i_ < s_.size()) {
        unsigned char d = static_cast<unsigned char>(s_[i_]);
        if (std::isalnum(d) || d == '_' || d == '/') ++i_; else break;
      }
      cur_.kind = Token::IDENT;
      cur_.text = s_.substr(b, i_ - b);
      return;
    }
    cur_.kind = Token::SYM;
    if (c == '-' && i_ + 1 < s_.size() && s_[i_ + 1] == '>') {
      cur_.text = "->";
      i_ += 2;
      return;
    }
    cur_.text = std::string(1, static_cast<char>(c));
    ++i_;
  }
  const std::string& s_;
  size_t i_ = 0;
  int line_ = 1;
  Token cur_;
};

// Parse-time expression with names still unresolved.
struct PNode {
  Expr::Kind kind = Expr::NIL;
  std::string a, b;
  int l = -1, r = -1;
};

struct PendingPerm {
  int slot;
  int root;
};
struct PendingAllowed {
  int slot;
  size_t cls;
  std::string rel;
};

}  // namespace

int Schema::name_id(const std::string& n) {
  for (size_t i = 0; i < names.size(); ++i)
    if (names[i] == n) return static_cast<int>(i);
  names.push_back(n);
  return static_cast<int>(names.size()) - 1;
}
int Schema::type_id(const std::string& n) const {
  for (size_t i = 0; i < types.size(); ++i)
    if (types[i].name == n) return static_cast<int>(i);
  return -1;
}
int Schema::slot_id(int type, const std::string& n) const {
  if (type < 0 || type >= static_cast<int>(types.size())) return -1;
  for (int s : types[type].slots)
    if (slots[s].name == n) return s;
  return -1;
}
int Schema::slot_by_name_id(int type, int nid) const {
  for (int s : types[type].slots)
    if (slots[s].name_id == nid) return s;
  return -1;
}
int Schema::class_of(int rel_slot, uint16_t stype, uint16_t sslot) const {
  const auto& cls = slots[rel_slot].classes;
  for (size_t k = 0; k < cls.size(); ++k)
    if (cls[k].stype == stype && cls[k].sslot == sslot) return static_cast<int>(k);
  return -1;
}

std::string Schema::parse(const std::string& text) {
  try {
    *this = Schema();
    // Pass 1: definition names, so subject types may be forward references.
    {
      Scanner sc(text);
      while (sc.peek().kind != Token::END) {
        if (sc.is_word("definition")) {
          sc.take();
          if (sc.peek().kind == Token::IDENT) {
            if (type_id(sc.peek().text) >= 0) sc.fail("duplicate definition");
            types.push_back(TypeInfo{sc.peek().text, {}});
          }
        } else {
          sc.take();
        }
      }
    }
    if (types.size() >= 0xFFF0) return "too many definitions";
    std::vector<PNode> pn;
    std::vector<PendingPerm> pperms;
    std::vector<PendingAllowed> pallowed;
    Scanner sc(text);

    // expression grammar: '+' binds tightest, then '&', then '-'; left associative
    std::function<int(int)> level;
    std::function<int()> primary = [&]() -> int {
      if (sc.is_sym("(")) {
        sc.take();
        int e = level(0);
        sc.expect_sym(")");
        return e;
      }
      if (sc.peek().kind != Token::IDENT) sc.fail("expected relation, permission, nil or '('");
      std::string a = sc.take().text;
      PNode n;
      if (a == "nil") {
        n.kind = Expr::NIL;
      } else if (sc.is_sym("->")) {
        sc.take();
        n.kind = Expr::ARROW;
        n.a = a;
        n.b = sc.expect_ident("permission name after '->'");
      } else if (sc.is_sym(".")) {
        sc.take();
        std::string fn = sc.expect_ident("'any'");
        if (fn != "any") sc.fail("only .any(...) arrows are supported");
        sc.expect_sym("(");
        n.kind = Expr::ARROW;
        n.a = a;
        n.b = sc.expect_ident("permission name");
        sc.expect_sym(")");
      } else {
        n.kind = Expr::REF;
        n.a = a;
      }
      pn.push_back(n);
      return static_cast<int>(pn.size()) - 1;
    };
    level = [&](int lvl) -> int {
      static const char* sym[3] = {"-", "&", "+"};
      static const Expr::Kind kind[3] = {Expr::EXCL, Expr::INTER, Expr::UNION};
      if (lvl == 3) return primary();
      int l = level(lvl + 1);
      while (sc.is_sym(sym[lvl])) {
        sc.take();
        int r = level(lvl + 1);
        PNode n;
        n.kind = kind[lvl];
        n.l = l;
        n.r = r;
        pn.push_back(n);
        l = static_cast<int>(pn.size()) - 1;
      }
      return l;
    };

    auto add_slot = [&](int type, const std::string& name, bool is_perm) -> int {
      if (slot_id(type, name) >= 0) sc.fail("duplicate relation or permission '" + name + "'");
      if (slots.size() >= 0xFFF0) sc.fail("too many relations/permissions");
      SlotInfo s;
      s.name = name;
      s.name_id = name_id(name);
      s.type = static_cast<uint16_t>(type);
      s.is_perm = is_perm;
      slots.push_back(s);
      types[type].slots.push_back(static_cast<int>(slots.size()) - 1);
      return static_cast<int>(slots.size()) - 1;
    };

    while (sc.peek().kind != Token::END) {
      if (sc.is_word("use")) {
        sc.take();
        if (sc.expect_ident("feature name") == "expiration") use_expiration = true;
        continue;
      }
      if (sc.is_word("caveat")) sc.fail("caveats are not supported");
      if (!sc.is_word("definition")) sc.fail("expected 'definition'");
      sc.take();
      int type = type_id(sc.expect_ident("definition name"));
      sc.expect_sym("{");
      while (!sc.is_sym("}")) {
        if (sc.is_word("relation")) {
          sc.take();
          int s = add_slot(type, sc.expect_ident("relation name"), false);
          sc.expect_sym(":");
          for (;;) {
            ClassInfo c{};
            int st = type_id(sc.expect_ident("subject type"));
            if (st < 0) sc.fail("unknown subject type");
            c.stype = static_cast<uint16_t>(st);
            c.sslot = kNone;
            std::string pending;
            if (sc.is_sym(":")) {
              sc.take();
              sc.expect_sym("*");
              c.sslot = kWildcard;
            } else if (sc.is_sym("#")) {
              sc.take();
              pending = sc.expect_ident("subject relation");
            }
            if (sc.is_word("with")) {
              sc.take();
              if (sc.expect_ident("'expiration'") != "expiration")
                sc.fail("caveats are not supported (only 'with expiration')");
              c.expiry = true;
            }
            slots[s].classes.push_back(c);
            if (!pending.empty()) pallowed.push_back({s, slots[s].classes.size() - 1, pending});
            if (!sc.is_sym("|")) break;
            sc.take();
          }
          if (slots[s].classes.size() > static_cast<size_t>(kMaxClasses))
            sc.fail("too many allowed subject kinds on one relation (max " + std::to_string(kMaxClasses) + ")");
        } else if (sc.is_word("permission")) {
          sc.take();
          int s = add_slot(type, sc.expect_ident("permission name"), true);
          sc.expect_sym("=");
          pperms.push_back({s, level(0)});
        } else {
          sc.fail("expected 'relation' or 'permission'");
        }
      }
      sc.expect_sym("}");
    }

    for (const auto& pa : pallowed) {
      ClassInfo& c = slots[pa.slot].classes[pa.cls];
      int sr = slot_id(c.stype, pa.rel);
      if (sr < 0)
        return "relation " + types[slots[pa.slot].type].name + "#" + slots[pa.slot].name + ": subject relation " +
               types[c.stype].name + "#" + pa.rel + " does not exist";
      c.sslot = static_cast<uint16_t>(sr);
    }
    // merge duplicate userset classes (e.g. listed twice)
    for (auto& s : slots) {
      std::vector<ClassInfo> uniq;
      for (const auto& c : s.classes) {
        bool dup = false;
        for (auto& u : uniq)
          if (u.stype == c.stype && u.sslot == c.sslot) {
            u.expiry = u.expiry || c.expiry;
            dup = true;
          }
        if (!dup) uniq.push_back(c);
      }
      s.classes = uniq;
    }

    // resolve permission expressions
    std::function<int(int, int)> resolve = [&](int type, int p) -> int {
      const PNode& n = pn[p];
      Expr e;
      e.kind = n.kind;
      switch (n.kind) {
        case Expr::NIL: break;
        case Expr::REF:
          e.slot = slot_id(type, n.a);
          if (e.slot < 0)
            throw std::runtime_error("definition " + types[type].name + ": unknown relation or permission '" + n.a + "'");
          break;
        case Expr::ARROW:
          e.slot = slot_id(type, n.a);
          if (e.slot < 0 || slots[e.slot].is_perm)
            throw std::runtime_error("definition " + types[type].name + ": arrow '" + n.a + "->" + n.b +
                                     "' needs a relation on the left");
          e.name = name_id(n.b);
          break;
        default:
          e.l = resolve(type, n.l);
          e.r = resolve(type, n.r);
      }
      exprs.push_back(e);
      return static_cast<int>(exprs.size()) - 1;
    };
    for (const auto& pp : pperms) slots[pp.slot].expr = resolve(slots[pp.slot].type, pp.root);
    return compile();
  } catch (const std::exception& ex) {
    return ex.what();
  }
}

// ---------------------------------------------------------------- compile

std::string Schema::compile() {
  // data relations and class tables
  rel_slots.clear();
  d_cls.clear();
  has_expiry = false;
  for (size_t s = 0; s < slots.size(); ++s)
    if (!slots[s].is_perm) {
      slots[s].rel_index = static_cast<int>(rel_slots.size());
      rel_slots.push_back(static_cast<int>(s));
      for (const auto& c : slots[s].classes) has_expiry = has_expiry || c.expiry;
    }

  struct UOp {
    int kind;  // OP_REL / OP_ARROW
    int rel_slot;
    int name;
    bool operator==(const UOp& o) const { return kind == o.kind && rel_slot == o.rel_slot && name == o.name; }
  };
  struct L {
    bool is_union = true;
    std::vector<UOp> ops;
    std::vector<int> members;
    TreeOpKind op = T_OR;
    int trivial_slot = -1;
    std::vector<L> kids;
  };
  std::vector<int> stack;  // permission slots being lowered (cycle detection)
  std::function<L(int)> lower_expr;
  std::function<L(int)> lower_slot = [&](int s) -> L {
    const SlotInfo& si = slots[s];
    if (!si.is_perm) {
      L u;
      u.ops.push_back({OP_REL, s, -1});
      u.members.push_back(s);
      return u;
    }
    if (std::find(stack.begin(), stack.end(), s) != stack.end())
      throw std::runtime_error("permission " + types[si.type].name + "#" + si.name +
                               " refers to itself on the same object (unsupported)");
    stack.push_back(s);
    L n = lower_expr(si.expr);
    stack.pop_back();
    if (n.is_union) {
      if (std::find(n.members.begin(), n.members.end(), s) == n.members.end()) n.members.push_back(s);
      return n;
    }
    L t;  // OR(TRIVIAL(s), tree): a userset subject type:obj#s is a member of itself
    t.is_union = false;
    t.op = T_OR;
    L triv;
    triv.is_union = false;
    triv.op = T_TRIVIAL;
    triv.trivial_slot = s;
    t.kids.push_back(triv);
    t.kids.push_back(n);
    return t;
  };
  lower_expr = [&](int e) -> L {
    const Expr& x = exprs[e];
    switch (x.kind) {
      case Expr::NIL: return L{};
      case Expr::REF: return lower_slot(x.slot);
      case Expr::ARROW: {
        L u;
        u.ops.push_back({OP_ARROW, x.slot, x.name});
        return u;
      }
      default: break;
    }
    L a = lower_expr(x.l), b = lower_expr(x.r);
    if (x.kind == Expr::UNION && a.is_union && b.is_union) {
      for (const auto& o : b.ops)
        if (std::find(a.ops.begin(), a.ops.end(), o) == a.ops.end()) a.ops.push_back(o);
      for (int m : b.members)
        if (std::find(a.members.begin(), a.members.end(), m) == a.members.end()) a.members.push_back(m);
      return a;
    }
    L t;
    t.is_union = false;
    t.op = x.kind == Expr::UNION ? T_OR : (x.kind == Expr::INTER ? T_AND : T_ANDNOT);
    t.kids.push_back(a);
    t.kids.push_back(b);
    return t;
  };

  d_slots.assign(slots.size(), DSlot{});
  d_units.clear();
  d_ops.clear();
  d_tgts.clear();
  d_members.clear();
  d_trees.clear();
  d_tree_ops.clear();
  d_leaf_units.clear();
  has_nonpure = false;
  max_leaves = 1;

  auto emit_unit = [&](const L& u) -> int {
    DUnit du{};
    du.op_begin = static_cast<uint16_t>(d_ops.size());
    for (const auto& o : u.ops) {
      DOp d{};
      d.kind = static_cast<uint16_t>(o.kind);
      d.rel = static_cast<uint16_t>(slots[o.rel_slot].rel_index);
      d.tgt_begin = static_cast<uint16_t>(d_tgts.size());
      if (o.kind == OP_ARROW) {
        for (const auto& c : slots[o.rel_slot].classes) {
          int tgt = c.sslot == kWildcard ? -1 : slot_by_name_id(c.stype, o.name);
          d_tgts.push_back(tgt < 0 ? kNone : static_cast<uint16_t>(tgt));
        }
      }
      d_ops.push_back(d);
    }
    du.op_end = static_cast<uint16_t>(d_ops.size());
    du.mem_begin = static_cast<uint16_t>(d_members.size());
    for (int m : u.members) d_members.push_back(static_cast<uint16_t>(m));
    du.mem_end = static_cast<uint16_t>(d_members.size());
    du.flags = 0;
    for (const auto& o : u.ops) {
      if (o.kind == OP_ARROW) du.flags |= UF_EXPANSIVE;
      for (const auto& c : slots[o.rel_slot].classes)
        if (c.sslot != kNone && c.sslot != kWildcard) du.flags |= UF_EXPANSIVE;
    }
    d_units.push_back(du);
    if (d_ops.size() > 0xFFF0 || d_tgts.size() > 0xFFF0 || d_members.size() > 0xFFF0 || d_units.size() > 0x7FF0)
      throw std::runtime_error("schema too large for the device program");
    return static_cast<int>(d_units.size()) - 1;
  };

  try {
    for (size_t s = 0; s < slots.size(); ++s) {
      L n = lower_slot(static_cast<int>(s));
      DSlot& ds = d_slots[s];
      ds.type = slots[s].type;
      if (n.is_union) {
        ds.kind = slots[s].is_perm ? SK_PURE : SK_RELATION;
        ds.unit = static_cast<uint16_t>(emit_unit(n));
        slots[s].kind = ds.kind;
        slots[s].unit = ds.unit;
      } else {
        has_nonpure = true;
        ds.kind = SK_NONPURE;
        DTree t{};
        t.op_begin = static_cast<uint16_t>(d_tree_ops.size());
        t.leaf_begin = static_cast<uint16_t>(d_leaf_units.size());
        uint16_t n_leaves = 0;
        int depth = 0, max_depth = 0;
        std::vector<const L*> seen_leaves;  // identical union groups share one leaf job
        std::function<void(const L&)> post = [&](const L& x) {
          if (x.is_union) {
            uint16_t idx = n_leaves;
            for (size_t i = 0; i < seen_leaves.size(); ++i)
              if (seen_leaves[i]->ops == x.ops && seen_leaves[i]->members == x.members) idx = static_cast<uint16_t>(i);
            if (idx == n_leaves) {
              seen_leaves.push_back(&x);
              d_leaf_units.push_back(static_cast<uint16_t>(emit_unit(x)));
              ++n_leaves;
            }
            d_tree_ops.push_back(DTreeOp{T_LEAF, idx});
            max_depth = std::max(max_depth, ++depth);
            return;
          }
          if (x.op == T_TRIVIAL) {
            d_tree_ops.push_back(DTreeOp{T_TRIVIAL, static_cast<uint16_t>(x.trivial_slot)});
            max_depth = std::max(max_depth, ++depth);
            return;
          }
          post(x.kids[0]);
          post(x.kids[1]);
          d_tree_ops.push_back(DTreeOp{static_cast<uint16_t>(x.op), 0});
          --depth;
        };
        post(n);
        t.op_end = static_cast<uint16_t>(d_tree_ops.size());
        t.n_leaves = n_leaves;
        for (uint16_t l = 0; l < n_leaves; ++l) t.flags |= d_units[d_leaf_units[t.leaf_begin + l]].flags & UF_EXPANSIVE;
        if (n_leaves > kMaxLeaves)
          throw std::runtime_error("permission " + types[slots[s].type].name + "#" + slots[s].name +
                                   " has too many union groups under & / - (max " + std::to_string(kMaxLeaves) + ")");
        if (max_depth > 32 || d_tree_ops.size() > 0xFFF0)
          throw std::runtime_error("permission " + types[slots[s].type].name + "#" + slots[s].name +
                                   " nests & / - too deeply for the device evaluator");
        max_leaves = std::max<uint32_t>(max_leaves, n_leaves);
        ds.unit = static_cast<uint16_t>(d_trees.size());
        d_trees.push_back(t);
        slots[s].kind = SK_NONPURE;
        slots[s].tree = ds.unit;
      }
    }
  } catch (const std::exception& ex) {
    return ex.what();
  }

  // A direct class is worth answering from the subject's reverse rows only when it is probed after a
  // fan-out, i.e. when some unit that contains its relation is the TARGET of a userset or arrow edge.
  // A class that is only ever probed at the root object of a check (pod#viewer@user in a flat schema,
  // document#banned@user) costs one forward binary search there; loading its reverse row at admission
  // would cost the same two sectors and fill the per-check set for nothing.
  std::vector<uint8_t> unit_pushed(d_units.size(), 0);
  {
    auto mark_slot = [&](uint16_t ts) {
      if (ts == kNone || ts >= d_slots.size()) return;
      if (d_slots[ts].kind == SK_NONPURE) {
        const DTree& t = d_trees[d_slots[ts].unit];
        for (uint16_t l = 0; l < t.n_leaves; ++l) unit_pushed[d_leaf_units[t.leaf_begin + l]] = 1;
      } else {
        unit_pushed[d_slots[ts].unit] = 1;
      }
    };
    for (const DUnit& u : d_units)
      for (int oi = u.op_begin; oi < u.op_end; ++oi) {
        const DOp& op = d_ops[oi];
        const auto& classes = slots[rel_slots[op.rel]].classes;
        for (size_t k = 0; k < classes.size(); ++k) {
          if (op.kind == OP_ARROW) mark_slot(d_tgts[op.tgt_begin + k]);
          else if (classes[k].sslot != kNone && classes[k].sslot != kWildcard) mark_slot(classes[k].sslot);
        }
      }
  }
  std::vector<uint8_t> rel_fanout(rel_slots.size(), 0);
  for (size_t u = 0; u < d_units.size(); ++u)
    if (unit_pushed[u])
      for (int oi = d_units[u].op_begin; oi < d_units[u].op_end; ++oi)
        if (d_ops[oi].kind == OP_REL) rel_fanout[d_ops[oi].rel] = 1;
  for (int rs : rel_slots)
    for (const auto& c : slots[rs].classes) {
      uint16_t fl = c.expiry ? CF_EXPIRY : 0;
      if (c.sslot == kNone && !c.expiry && rel_fanout[slots[rs].rel_index]) fl |= CF_INVERT;
      d_cls.push_back(DCls{c.stype, c.sslot, fl, static_cast<uint16_t>(slots[rs].rel_index), 0, slots[rs].type, 0, 0});
    }
  d_type_inv.assign(types.size(), DTypeInv{0, 0});
  d_inv_cls.clear();
  for (size_t t = 0; t < types.size(); ++t) {
    d_type_inv[t].begin = static_cast<uint16_t>(d_inv_cls.size());
    for (size_t c = 0; c < d_cls.size(); ++c)
      if ((d_cls[c].flags & CF_INVERT) && d_cls[c].stype == t) d_inv_cls.push_back(static_cast<uint16_t>(c));
    d_type_inv[t].end = static_cast<uint16_t>(d_inv_cls.size());
  }
  d_type_rcls.assign(types.size(), DTypeInv{0, 0});
  d_rcls.clear();
  for (size_t t = 0; t < types.size(); ++t) {
    d_type_rcls[t].begin = static_cast<uint16_t>(d_rcls.size());
    for (size_t c = 0; c < d_cls.size(); ++c)
      if (d_cls[c].stype == t) d_rcls.push_back(static_cast<uint16_t>(c));
    d_type_rcls[t].end = static_cast<uint16_t>(d_rcls.size());
  }
  compute_forward_masks();
  compute_expand_templates();
  return "";
}

// The tree of Expand(T:r, P) restricted to what r's own rows decide (DESIGN.md §2, "ExpandPermissionTree"): a chain of
// + or & is one n-ary node, - stays binary, a bare operand is a one-child union, a same-object reference is the
// referenced slot's subtree and an arrow is a node whose children the next level expands.
void Schema::compute_expand_templates() {
  const size_t ns = slots.size();
  x_nodes.clear();
  x_tgts.clear();
  x_counted.clear();
  x_root.assign(ns, kNoTemplate);
  x_ok.assign(ns, 0);
  for (size_t s = 0; s < ns; ++s) {
    std::vector<XNode> t;
    std::vector<uint8_t> kids;
    std::vector<std::vector<uint32_t>> tgts;  // per node: the arrow's target slot per class
    bool over = false;
    auto add = [&](uint16_t op, int slot, int parent) -> int {
      if (t.size() >= static_cast<size_t>(kMaxExpandTemplate)) {
        over = true;
        return -1;
      }
      XNode n{};
      n.op = op;
      n.slot = static_cast<uint16_t>(slot);
      if (parent >= 0) {
        n.parent = static_cast<uint8_t>(parent);
        n.rank = kids[parent]++;
      }
      t.push_back(n);
      kids.push_back(0);
      tgts.emplace_back();
      return static_cast<int>(t.size()) - 1;
    };
    std::function<void(int, int)> of_slot;
    std::function<void(int, int, int)> of_expr, operand;
    auto flatten = [&](int e, Expr::Kind k, std::vector<int>* out) {
      std::function<void(int)> go = [&](int x) {
        if (exprs[x].kind == k) {
          go(exprs[x].l);
          go(exprs[x].r);
        } else {
          out->push_back(x);
        }
      };
      go(e);
    };
    of_slot = [&](int slot, int parent) {
      if (over) return;
      const SlotInfo& si = slots[slot];
      if (!si.is_perm) {
        const int n = add(X_REL, slot, parent);
        if (n >= 0) t[n].rel = static_cast<uint16_t>(si.rel_index);
        return;
      }
      of_expr(si.expr, slot, parent);
    };
    of_expr = [&](int e, int at, int parent) {
      if (over) return;
      const Expr& x = exprs[e];
      if (x.kind == Expr::UNION || x.kind == Expr::INTER) {
        const int n = add(x.kind == Expr::UNION ? X_UNION : X_INTER, at, parent);
        std::vector<int> ops;
        flatten(e, x.kind, &ops);
        for (int o : ops) operand(o, at, n);
      } else if (x.kind == Expr::EXCL) {
        const int n = add(X_EXCL, at, parent);
        operand(x.l, at, n);
        operand(x.r, at, n);
      } else {
        operand(e, at, add(X_UNION, at, parent));
      }
    };
    operand = [&](int e, int at, int parent) {
      if (over) return;
      const Expr& x = exprs[e];
      switch (x.kind) {
        case Expr::REF: of_slot(x.slot, parent); break;
        case Expr::NIL: add(X_NIL, at, parent); break;
        case Expr::ARROW: {
          const int n = add(X_ARROW, at, parent);
          if (n < 0) return;
          t[n].rel = static_cast<uint16_t>(slots[x.slot].rel_index);
          for (const ClassInfo& c : slots[x.slot].classes) {
            const int target = c.sslot == kWildcard ? -1 : slot_by_name_id(c.stype, x.name);
            tgts[n].push_back(target < 0 ? kNoTemplate : static_cast<uint32_t>(target));
          }
          break;
        }
        default: of_expr(e, at, parent);
      }
    };
    of_slot(static_cast<int>(s), -1);
    if (over) continue;
    const uint32_t base = static_cast<uint32_t>(x_nodes.size());
    t[0].size = static_cast<uint8_t>(t.size());
    t[0].counted = static_cast<uint32_t>(x_counted.size());
    for (size_t i = 0; i < t.size(); ++i) {
      if (t[i].op == X_REL || t[i].op == X_ARROW) {
        t[i].count = t[0].ncount++;
        x_counted.push_back(static_cast<uint32_t>(i));
      }
      if (t[i].op == X_ARROW) {
        t[i].tgt = static_cast<uint32_t>(x_tgts.size());
        x_tgts.insert(x_tgts.end(), tgts[i].begin(), tgts[i].end());  // slots for now: roots below
      }
    }
    x_nodes.insert(x_nodes.end(), t.begin(), t.end());
    x_root[s] = base;
    x_ok[s] = 1;
  }
  // a slot is expandable when its template and every template its arrows reach fit
  for (bool changed = true; changed;) {
    changed = false;
    for (size_t s = 0; s < ns; ++s) {
      if (!x_ok[s]) continue;
      const XNode* t = x_nodes.data() + x_root[s];
      for (uint32_t i = 0; i < t[0].size && x_ok[s]; ++i) {
        if (t[i].op != X_ARROW) continue;
        for (size_t k = 0; k < slots[rel_slots[t[i].rel]].classes.size(); ++k) {
          const uint32_t target = x_tgts[t[i].tgt + k];
          if (target != kNoTemplate && !x_ok[target]) {
            x_ok[s] = 0;
            changed = true;
            break;
          }
        }
      }
    }
  }
  for (XNode& n : x_nodes) {
    if (n.op != X_ARROW) continue;
    for (size_t k = 0; k < slots[rel_slots[n.rel]].classes.size(); ++k) {
      uint32_t& target = x_tgts[n.tgt + k];
      if (target != kNoTemplate) target = x_root[target];
    }
  }
}

void Schema::compute_forward_masks() {
  std::vector<uint32_t> cls_begin(rel_slots.size() + 1, 0);
  for (size_t r = 0; r < rel_slots.size(); ++r)
    cls_begin[r + 1] = cls_begin[r] + static_cast<uint32_t>(slots[rel_slots[r]].classes.size());
  fwd_mask_words = std::max<uint32_t>(1, (cls_begin.back() + 31) / 32);
  fwd_mask.assign(slots.size() * fwd_mask_words, 0);
  for (size_t s = 0; s < slots.size(); ++s) {
    uint32_t* m = fwd_mask.data() + s * fwd_mask_words;
    std::vector<uint8_t> seen(slots.size(), 0);
    std::vector<uint16_t> todo{static_cast<uint16_t>(s)};
    while (!todo.empty()) {
      const uint16_t x = todo.back();
      todo.pop_back();
      if (x >= slots.size() || seen[x]) continue;
      seen[x] = 1;
      std::vector<uint16_t> units;
      if (d_slots[x].kind == SK_NONPURE) {
        const DTree& t = d_trees[d_slots[x].unit];
        for (uint16_t l = 0; l < t.n_leaves; ++l) units.push_back(d_leaf_units[t.leaf_begin + l]);
      } else {
        units.push_back(d_slots[x].unit);
      }
      for (uint16_t u : units)
        for (int oi = d_units[u].op_begin; oi < d_units[u].op_end; ++oi) {
          const DOp& op = d_ops[oi];
          const auto& classes = slots[rel_slots[op.rel]].classes;
          for (size_t k = 0; k < classes.size(); ++k) {
            if (classes[k].sslot == kWildcard) continue;
            const uint32_t gc = cls_begin[op.rel] + static_cast<uint32_t>(k);
            m[gc >> 5] |= 1u << (gc & 31);
            if (op.kind == OP_ARROW) todo.push_back(d_tgts[op.tgt_begin + k]);
            else if (classes[k].sslot != kNone) todo.push_back(classes[k].sslot);
          }
        }
    }
  }
}

void Schema::forward_tables(const std::vector<DRel>& rels, std::vector<FwdClass>* fwd, std::vector<uint32_t>* type_off) const {
  fwd->clear();
  type_off->assign(types.size() + 1, 0);
  for (size_t t = 0; t < types.size(); ++t) {
    (*type_off)[t] = static_cast<uint32_t>(fwd->size());
    for (size_t r = 0; r < rels.size() && r < rel_slots.size(); ++r) {
      if (slots[rel_slots[r]].type != t) continue;
      const DRel& d = rels[r];
      for (uint16_t k = 0; k < d.ncls; ++k) {
        const uint16_t gc = static_cast<uint16_t>(d.cls_begin + k);
        if (d_cls[gc].sslot == kWildcard) continue;
        FwdClass f{};
        f.row_base = d.row_base + k;
        f.nres = d.nres;
        f.ncls = static_cast<uint16_t>(d.stride);
        f.stype = d_cls[gc].stype;
        f.gc = gc;
        fwd->push_back(f);
      }
    }
  }
  (*type_off)[types.size()] = static_cast<uint32_t>(fwd->size());
}

std::vector<uint8_t> Schema::blob(const std::vector<DRel>& rels, const std::vector<DCls>& cls) const {
  DHeader h{};
  h.magic = 0x5A47504Du;  // "ZGPM"
  h.n_types = static_cast<uint32_t>(types.size());
  h.n_slots = static_cast<uint32_t>(d_slots.size());
  h.n_units = static_cast<uint32_t>(d_units.size());
  h.n_ops = static_cast<uint32_t>(d_ops.size());
  h.n_rels = static_cast<uint32_t>(rels.size());
  h.n_cls = static_cast<uint32_t>(d_cls.size());
  h.n_trees = static_cast<uint32_t>(d_trees.size());
  h.n_tree_ops = static_cast<uint32_t>(d_tree_ops.size());
  h.max_leaves = max_leaves;
  h.has_nonpure = has_nonpure;
  h.has_expiry = has_expiry;
  h.reach_words = 0;
  std::vector<uint8_t> out(sizeof(DHeader));
  auto put = [&](const void* p, size_t bytes, uint32_t* off) {
    size_t at = (out.size() + 15) & ~size_t(15);
    out.resize(at + bytes);
    if (bytes) std::memcpy(out.data() + at, p, bytes);
    *off = static_cast<uint32_t>(at);
  };
  // flatten every unit into steps for THIS snapshot (empty classes vanish)
  std::vector<DUnit> units = d_units;
  std::vector<DStep> steps;
  for (auto& u : units) {
    u.step_begin = static_cast<uint16_t>(steps.size());
    for (int oi = u.op_begin; oi < u.op_end; ++oi) {
      const DOp& op = d_ops[oi];
      const DRel& r = rels[op.rel];
      for (uint16_t k = 0; k < r.ncls; ++k) {
        const DCls& c = cls[r.cls_begin + k];
        if (c.flags & CF_EMPTY) continue;
        DStep st{};
        st.row_base = r.row_base + k;
        st.nres = r.nres;
        st.ncls = static_cast<uint16_t>(r.stride);
        st.flags = c.flags;
        st.gc = static_cast<uint16_t>(r.cls_begin + k);
        st.stype = c.stype;
        st.tslot = kNone;
        if (op.kind == OP_REL) {
          if (c.sslot == kNone) st.kind = ST_DIRECT;
          else if (c.sslot == kWildcard) st.kind = ST_WILD;
          else {
            st.kind = ST_PUSH;
            st.tslot = c.sslot;
          }
        } else {
          st.kind = ST_PUSH;
          st.tslot = d_tgts[op.tgt_begin + k];
          if (st.tslot == kNone) continue;
        }
        steps.push_back(st);
      }
    }
    u.step_end = static_cast<uint16_t>(steps.size());
    // probes (answered by the lane on its own) before the edge classes that push ranges (warp-collective)
    std::stable_partition(steps.begin() + u.step_begin, steps.end(), [](const DStep& x) { return x.kind != ST_PUSH; });
    u.push_begin = u.step_begin;
    while (u.push_begin < u.step_end && steps[u.push_begin].kind != ST_PUSH) ++u.push_begin;
    bool leaf = u.step_end > u.step_begin;
    for (int i = u.step_begin; i < u.step_end; ++i)
      leaf = leaf && steps[i].kind == ST_DIRECT && (steps[i].flags & CF_INVERT);
    if (leaf) u.flags |= UF_LEAF_INV;
  }
  std::vector<uint16_t> inv_pos(cls.size(), kNone);  // class -> index in its type's invertible list
  for (const auto& ti : d_type_inv)
    for (uint16_t i = ti.begin; i < ti.end; ++i) inv_pos[d_inv_cls[i]] = static_cast<uint16_t>(i - ti.begin);
  for (auto& st : steps) {
    st.tinv = st.kind == ST_DIRECT ? inv_pos[st.gc] : kNone;
    if (st.kind != ST_PUSH) continue;
    st.tunit = kNone;
    st.tgc = kNone;
    if (d_slots[st.tslot].kind == SK_NONPURE) continue;
    st.tunit = d_slots[st.tslot].unit;
    const DUnit& tu = units[st.tunit];
    if ((tu.flags & UF_LEAF_INV) && tu.step_end - tu.step_begin == 1) {
      st.flags |= kStepTargetLeaf;
      st.tgc = steps[tu.step_begin].gc;
      st.tinv = inv_pos[st.tgc];
      st.tstype = steps[tu.step_begin].stype;
    }
  }
  // second level: the target unit is one userset class whose children are leaf visits
  for (auto& st : steps) {
    if (st.kind != ST_PUSH || st.tunit == kNone || (st.flags & (kStepTargetLeaf | CF_EXPIRY))) continue;
    const DUnit& tu = units[st.tunit];
    if (tu.step_end - tu.step_begin != 1) continue;
    const DStep& in = steps[tu.step_begin];
    if (in.kind != ST_PUSH || !(in.flags & kStepTargetLeaf) || (in.flags & CF_EXPIRY)) continue;
    st.flags |= kStepTargetL2;
    st.tgc = in.gc;
    st.tinv = in.tinv;
    st.tstype = in.tstype;
  }
  h.n_steps = static_cast<uint32_t>(steps.size());
  // (rels / ops / tgts stay on the host: the kernels only read the flattened steps)
  h.off_rels = h.off_ops = h.off_tgts = 0;
  put(steps.data(), steps.size() * sizeof(DStep), &h.off_steps);
  put(cls.data(), cls.size() * sizeof(DCls), &h.off_cls);  // 8-byte aligned members
  put(d_slots.data(), d_slots.size() * sizeof(DSlot), &h.off_slots);
  put(units.data(), units.size() * sizeof(DUnit), &h.off_units);
  put(d_members.data(), d_members.size() * 2, &h.off_members);
  put(d_trees.data(), d_trees.size() * sizeof(DTree), &h.off_trees);
  put(d_tree_ops.data(), d_tree_ops.size() * sizeof(DTreeOp), &h.off_tree_ops);
  put(d_leaf_units.data(), d_leaf_units.size() * 2, &h.off_leaf_units);
  put(d_type_inv.data(), d_type_inv.size() * sizeof(DTypeInv), &h.off_type_inv);
  put(d_inv_cls.data(), d_inv_cls.size() * 2, &h.off_inv_cls);
  put(d_type_rcls.data(), d_type_rcls.size() * sizeof(DTypeInv), &h.off_type_rcls);
  put(d_rcls.data(), d_rcls.size() * 2, &h.off_rcls);
  h.off_reach = 0;
  out.resize((out.size() + 15) & ~size_t(15));
  h.total_bytes = static_cast<uint32_t>(out.size());
  std::memcpy(out.data(), &h, sizeof h);
  return out;
}

int mark_rsetless_slots(std::vector<uint8_t>* blob, const std::vector<uint16_t>& indexed_tgc) {
  uint8_t* const b = blob->data();
  const DHeader* h = reinterpret_cast<const DHeader*>(b);
  DSlot* slots = reinterpret_cast<DSlot*>(b + h->off_slots);
  const DUnit* units = reinterpret_cast<const DUnit*>(b + h->off_units);
  const DStep* steps = reinterpret_cast<const DStep*>(b + h->off_steps);
  const DTree* trees = reinterpret_cast<const DTree*>(b + h->off_trees);
  const uint16_t* leaf_units = reinterpret_cast<const uint16_t*>(b + h->off_leaf_units);
  auto unit_ok = [&](uint16_t u) {
    const DUnit& x = units[u];
    for (int i = x.step_begin; i < x.push_begin; ++i)
      if (steps[i].kind == ST_DIRECT && (steps[i].flags & CF_INVERT)) return false;
    for (int i = x.push_begin; i < x.step_end; ++i)
      if (!(steps[i].flags & kStepTargetL2) ||
          std::find(indexed_tgc.begin(), indexed_tgc.end(), steps[i].tgc) == indexed_tgc.end())
        return false;
    return true;
  };
  int marked = 0;
  for (uint32_t s = 0; s < h->n_slots; ++s) {
    bool ok = true;
    if (slots[s].kind == SK_NONPURE) {
      const DTree& t = trees[slots[s].unit];
      for (uint16_t l = 0; l < t.n_leaves && ok; ++l) ok = unit_ok(leaf_units[t.leaf_begin + l]);
    } else {
      ok = unit_ok(slots[s].unit);
    }
    slots[s].flags = static_cast<uint16_t>(ok ? slots[s].flags | SF_NO_RSET : slots[s].flags & ~SF_NO_RSET);
    marked += ok;
  }
  return marked;
}

int mark_flat_slots(std::vector<uint8_t>* blob, const std::vector<uint16_t>& tabled_tgc) {
  uint8_t* const b = blob->data();
  const DHeader* h = reinterpret_cast<const DHeader*>(b);
  DSlot* slots = reinterpret_cast<DSlot*>(b + h->off_slots);
  const DUnit* units = reinterpret_cast<const DUnit*>(b + h->off_units);
  const DStep* steps = reinterpret_cast<const DStep*>(b + h->off_steps);
  const DTypeInv* type_inv = reinterpret_cast<const DTypeInv*>(b + h->off_type_inv);
  int marked = 0;
  for (uint32_t s = 0; s < h->n_slots; ++s) {
    bool ok = slots[s].kind != SK_NONPURE && (slots[s].flags & SF_NO_RSET) && !tabled_tgc.empty();
    if (ok) {
      const DUnit& u = units[slots[s].unit];
      const int npush = u.step_end - u.push_begin;
      ok = npush >= 1 && npush <= kFlatSteps;
      for (int i = u.push_begin; i < u.step_end && ok; ++i)
        ok = std::find(tabled_tgc.begin(), tabled_tgc.end(), steps[i].tgc) != tabled_tgc.end() &&
             type_inv[steps[i].tstype].end - type_inv[steps[i].tstype].begin <= kMaxInvClasses;
    }
    slots[s].flags = static_cast<uint16_t>(ok ? slots[s].flags | SF_FLAT : slots[s].flags & ~SF_FLAT);
    marked += ok;
  }
  return marked;
}

}  // namespace zg
