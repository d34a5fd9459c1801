// regex.h — regex queries on the host: the pattern of a QueryAst `regex` leaf (quickwit-query
// query_ast/regex_query.rs -> tantivy_fst::Regex + AutomatonWeight) parsed and compiled to an automaton over Unicode
// code points, then run over a field's sorted term dictionary. The terms that match the WHOLE term (the automaton is
// anchored at both ends) are the query's expansions; the device unions their postings (QW_NODE_TERM_SET).
//
// Served exactly, or refused. The subset below is the one whose match set is known to equal the reference's:
//   literals (escaped metacharacters, \n \t \r \f \v \a \xHH \x{H...}, any UTF-8 code point), `.`, bracket classes
//   (ranges, negation, nested classes, escapes, ASCII POSIX classes), `|`, groups `( )` `(?: )` `(?P<n> )` `(?<n> )`,
//   greedy `* + ? {n} {n,} {n,m}`, flags i / s / m (set or cleared, scoped or global; `m` only affects anchors).
//   Perl classes \d \s \w (and negations) are served with their ASCII restriction [0-9], [\t\n\v\f\r ], [0-9A-Za-z_];
//   the reference's definitions are Unicode, so a walk that tests one against a non-ASCII code point refuses the split.
//   (?i) folds ASCII letters, plus the two orbits that leave ASCII: {k, K, U+212A KELVIN SIGN}, {s, S, U+017F LONG S};
//   a non-ASCII literal or class range under (?i) is refused (no Unicode case-folding tables here).
// Refused with QWGPU_EINVALID_QUERY ("failed to parse regex"), as the reference fails: syntax errors, look-around,
// back-references, zero-width assertions (^ $ \A \z \b \B: tantivy-fst rejects every one).
// Refused with QWGPU_EUNSUPPORTED: lazy repetitions and (?U), \p{..} / \P{..}, (?-u), (?x), escapes whose meaning
// differs between regex-syntax versions, class set operations (&& -- ~~), and an automaton of more than
// MAX_STATES states (or a walk that builds more than MAX_DFA_STATES automaton states, or whose automaton states hold
// more than MAX_DFA_ENTRIES NFA states together).
#pragma once
#include <algorithm>
#include <cctype>
#include <map>
#include <string>
#include <unordered_map>
#include <vector>

#include "common.h"

namespace qw {
namespace rx {

// NFA states after counted repetitions are expanded, the final state included (`x{9999}` takes 10 000). Above it the
// pattern is refused.
static const uint32_t MAX_STATES = 10000;
// distinct automaton states (sets of NFA states) one dictionary walk may build
static const uint32_t MAX_DFA_STATES = 1u << 16;
// NFA states held by all of those automaton states together (4 bytes each): bounds the walk's memory at about 64 MiB
static const uint32_t MAX_DFA_ENTRIES = 1u << 24;
static const uint32_t MAX_CP = 0x10FFFF;
static const uint32_t KELVIN = 0x212A, LONG_S = 0x17F;

[[noreturn]] inline void syntax(const char* what) { fail(QWGPU_EINVALID_QUERY, "invalid query: failed to parse regex: %s", what); }
[[noreturn]] inline void unsupported(const char* what) { fail(QWGPU_EUNSUPPORTED, "regex %s is not implemented on the GPU path", what); }

struct Range { uint32_t lo, hi; };
// a set of code points: sorted, disjoint, non-adjacent ranges. perl: holds a Perl class (\d \s \w or a negation)
struct Set {
  std::vector<Range> r;
  bool perl = false;
  void add(uint32_t lo, uint32_t hi) { r.push_back({lo, hi}); }
  void norm() {
    std::sort(r.begin(), r.end(), [](const Range& a, const Range& b) { return a.lo < b.lo; });
    std::vector<Range> o;
    for (const Range& x : r) {
      if (!o.empty() && x.lo <= o.back().hi + 1) o.back().hi = std::max(o.back().hi, x.hi);
      else o.push_back(x);
    }
    r.swap(o);
  }
  void negate() {
    norm();
    std::vector<Range> o;
    uint32_t next = 0;
    for (const Range& x : r) {
      if (x.lo > next) o.push_back({next, x.lo - 1});
      next = x.hi + 1;
    }
    if (next <= MAX_CP) o.push_back({next, MAX_CP});
    r.swap(o);
  }
  void merge(const Set& s) { r.insert(r.end(), s.r.begin(), s.r.end()); perl |= s.perl; }
  bool has(uint32_t c) const {
    size_t lo = 0, hi = r.size();
    while (lo < hi) {
      const size_t mid = (lo + hi) / 2;
      if (r[mid].hi < c) lo = mid + 1; else hi = mid;
    }
    return lo < r.size() && r[lo].lo <= c;
  }
  // (?i): ASCII letters fold in pairs; k and s also reach U+212A and U+017F
  void fold() {
    const std::vector<Range> in = r;
    for (const Range& x : in) {
      if (x.hi >= 0x80) unsupported("case-insensitive matching of non-ASCII characters");
      auto overlap = [&](uint32_t a, uint32_t b) { return x.lo <= b && a <= x.hi; };
      if (overlap('A', 'Z')) add(std::max<uint32_t>(x.lo, 'A') + 32, std::min<uint32_t>(x.hi, 'Z') + 32);
      if (overlap('a', 'z')) add(std::max<uint32_t>(x.lo, 'a') - 32, std::min<uint32_t>(x.hi, 'z') - 32);
      if (overlap('k', 'k') || overlap('K', 'K')) add(KELVIN, KELVIN);
      if (overlap('s', 's') || overlap('S', 'S')) add(LONG_S, LONG_S);
    }
    norm();
  }
};

struct Node {
  enum Kind { Empty, Chars, Cat, Alt, Rep } kind = Empty;
  Set set;                // Chars
  std::vector<Node> kids;  // Cat / Alt / Rep (one)
  uint32_t min = 0, max = 0;  // Rep; max == UINT32_MAX: unbounded
};

struct Flags { bool i = false, s = false; };

class Parser {
 public:
  explicit Parser(const std::string& p) : p_(p) {}
  Node parse() {
    Flags f;
    Node n = alt(f, 0);
    if (pos_ < p_.size()) syntax("unopened group");  // (alt stops at `)` only)
    return n;
  }

 private:
  const std::string& p_;
  size_t pos_ = 0;
  std::vector<std::string> names_;

  bool eof() const { return pos_ >= p_.size(); }
  char peek(size_t k = 0) const { return pos_ + k < p_.size() ? p_[pos_ + k] : '\0'; }
  uint32_t next_cp() {  // one UTF-8 code point of the pattern
    const unsigned char c = (unsigned char)p_[pos_];
    uint32_t n = c < 0x80 ? 1 : (c >> 5) == 6 ? 2 : (c >> 4) == 14 ? 3 : (c >> 3) == 30 ? 4 : 0;
    if (n == 0 || pos_ + n > p_.size()) syntax("invalid UTF-8 in the pattern");
    uint32_t cp = n == 1 ? c : n == 2 ? (c & 0x1F) : n == 3 ? (c & 0x0F) : (c & 0x07);
    for (uint32_t k = 1; k < n; k++) cp = (cp << 6) | ((unsigned char)p_[pos_ + k] & 0x3F);
    pos_ += n;
    return cp;
  }
  static Node chars(Set s) { Node n; n.kind = Node::Chars; n.set = std::move(s); return n; }
  static Set literal(uint32_t cp, const Flags& f) {
    Set s;
    s.add(cp, cp);
    if (f.i) s.fold();
    return s;
  }

  Node alt(Flags& f, int depth) {
    if (depth > 250) syntax("nesting limit exceeded");
    Node a;
    a.kind = Node::Alt;
    Node cat;
    cat.kind = Node::Cat;
    bool atom = false;  // the last item of the concatenation can take a repetition
    while (!eof() && peek() != ')') {
      const char c = peek();
      if (c == '|') {
        pos_++;
        a.kids.push_back(std::move(cat));
        cat = Node();
        cat.kind = Node::Cat;
        atom = false;
      } else if (c == '*' || c == '+' || c == '?' || c == '{') {
        if (!atom) syntax("repetition operator missing expression");
        Node& last = cat.kids.back();
        if (last.kind == Node::Rep) unsupported("repetition of a repetition");
        Node r;
        r.kind = Node::Rep;
        if (c == '{') counted(r);
        else {
          pos_++;
          r.min = c == '+' ? 1 : 0;
          r.max = c == '?' ? 1 : UINT32_MAX;
        }
        if (peek() == '?') unsupported("lazy repetition");
        if (peek() == '+') unsupported("repetition of a repetition");
        r.kids.push_back(std::move(last));
        last = std::move(r);
      } else if (c == '(') {
        pos_++;
        Node g;
        if (group(f, depth, &g)) { cat.kids.push_back(std::move(g)); atom = true; }
        else atom = false;  // a flag setting `(?i)`
      } else if (c == '[') {
        pos_++;
        cat.kids.push_back(chars(cls(f)));
        atom = true;
      } else if (c == '.') {
        pos_++;
        Set s;
        if (f.s) s.add(0, MAX_CP);
        else { s.add(0, '\n' - 1); s.add('\n' + 1, MAX_CP); }
        cat.kids.push_back(chars(s));
        atom = true;
      } else if (c == '^' || c == '$') {
        syntax("zero-width assertions are not supported");
      } else if (c == '\\') {
        pos_++;
        Set s;
        if (!escape(&s)) s = literal(s.r[0].lo, f);
        cat.kids.push_back(chars(s));
        atom = true;
      } else {
        cat.kids.push_back(chars(literal(next_cp(), f)));
        atom = true;
      }
    }
    a.kids.push_back(std::move(cat));
    return a;
  }

  uint32_t decimal() {
    if (!(peek() >= '0' && peek() <= '9')) {
      if (peek() == ' ') unsupported("counted repetition with spaces");
      syntax("invalid counted repetition");
    }
    uint64_t v = 0;
    while (peek() >= '0' && peek() <= '9') {
      v = v * 10 + (uint64_t)(peek() - '0');
      if (v > UINT32_MAX - 1) syntax("counted repetition too large");
      pos_++;
    }
    return (uint32_t)v;
  }
  void counted(Node& r) {
    pos_++;  // `{`
    if (peek() == ',') unsupported("counted repetition without a minimum");
    r.min = decimal();
    r.max = r.min;
    if (peek() == ',') {
      pos_++;
      r.max = peek() == '}' ? UINT32_MAX : decimal();
    }
    if (peek() != '}') syntax(eof() ? "unclosed counted repetition" : "invalid counted repetition");
    pos_++;
    if (r.min > r.max) syntax("invalid counted repetition range");
  }

  // after `(`: a group (true, *out set) or a flag setting for the rest of the enclosing group (false)
  bool group(Flags& f, int depth, Node* out) {
    Flags g = f;
    if (peek() == '?') {
      pos_++;
      if (peek() == '=' || peek() == '!') syntax("look-around is not supported");
      if (peek() == '<' && (peek(1) == '=' || peek(1) == '!')) syntax("look-around is not supported");
      if (peek() == 'P' && (peek(1) == '=' || peek(1) == '>')) syntax("backreferences are not supported");
      if (peek() == 'P' && peek(1) == '<') { pos_ += 2; name(); }
      else if (peek() == '<') { pos_++; name(); }
      else if (peek() == ':') pos_++;
      else {
        bool neg = false, any = false, after_neg = false;
        std::string seen;
        while (!eof() && peek() != ':' && peek() != ')') {
          const char c = p_[pos_++];
          if (c == '-') {
            if (neg) syntax("repeated flag negation");
            neg = true;
            after_neg = false;
            continue;
          }
          if (seen.find(c) != std::string::npos) syntax("duplicate flag");
          seen += c;
          any = true;
          after_neg = true;
          switch (c) {
            case 'i': g.i = !neg; break;
            case 's': g.s = !neg; break;
            case 'm': break;  // only changes what ^ and $ match, and anchors are refused
            case 'u': if (neg) unsupported("(?-u) (byte-oriented matching)"); break;
            case 'U': unsupported("(?U) (lazy repetitions)");
            case 'x': unsupported("(?x) (verbose mode)");
            case 'R': unsupported("(?R) (CRLF mode)");
            default: syntax("unrecognized flag");
          }
        }
        if (eof()) syntax("unclosed group");
        if (!any || (neg && !after_neg)) syntax("flag negation without a flag");
        if (p_[pos_++] == ')') { f = g; return false; }
      }
    }
    *out = alt(g, depth + 1);
    if (eof()) syntax("unclosed group");
    pos_++;  // `)`
    return true;
  }
  void name() {
    const size_t start = pos_;
    while (!eof() && peek() != '>') {
      const char c = peek();
      const bool ok = c == '_' || (c >= 'a' && c <= 'z') || (c >= 'A' && c <= 'Z') ||
                      (pos_ > start && ((c >= '0' && c <= '9') || c == '.' || c == '[' || c == ']'));
      if (!ok) syntax("invalid capture group name");
      pos_++;
    }
    if (eof() || pos_ == start) syntax("invalid capture group name");
    const std::string n = p_.substr(start, pos_ - start);
    if (std::find(names_.begin(), names_.end(), n) != names_.end()) syntax("duplicate capture group name");
    names_.push_back(n);
    pos_++;  // `>`
  }

  // after `\`: a class (true) or one literal code point in s->r[0] (false, not case-folded)
  bool escape(Set* s) {
    if (eof()) syntax("incomplete escape sequence");
    const unsigned char c = (unsigned char)peek();
    if (c >= 0x80) unsupported("escape of a non-ASCII character");
    pos_++;
    auto lit = [&](uint32_t cp) { s->add(cp, cp); return false; };
    switch (c) {
      case 'n': return lit('\n');
      case 't': return lit('\t');
      case 'r': return lit('\r');
      case 'f': return lit('\f');
      case 'v': return lit('\v');
      case 'a': return lit(7);
      case 'x': return lit(hex());
      case 'd': case 'D': case 's': case 'S': case 'w': case 'W': {
        const char k = (char)(c | 0x20);
        if (k == 'd') s->add('0', '9');
        else if (k == 's') { s->add('\t', '\r'); s->add(' ', ' '); }
        else { s->add('0', '9'); s->add('A', 'Z'); s->add('_', '_'); s->add('a', 'z'); }
        s->norm();
        if (c != k) s->negate();
        s->perl = true;
        return true;
      }
      case 'p': case 'P': unsupported("Unicode class (\\p / \\P)");
      case 'u': case 'U': unsupported("escape \\u / \\U");
      case 'b': case 'B': case 'A': case 'z': case '<': case '>':
        syntax("zero-width assertions are not supported");
      default: break;
    }
    if (c >= '0' && c <= '9') syntax("backreferences are not supported");
    if (c && strchr(".+*?()|[]{}^$#&-~\\", (int)c)) return lit(c);
    if (isalpha(c)) syntax("unrecognized escape sequence");
    unsupported("escape of a character that is not a metacharacter");
  }
  uint32_t hex() {
    uint32_t v = 0;
    auto digit = [&](char c) -> int { return c >= '0' && c <= '9' ? c - '0' : c >= 'a' && c <= 'f' ? c - 'a' + 10 : c >= 'A' && c <= 'F' ? c - 'A' + 10 : -1; };
    if (peek() == '{') {
      pos_++;
      int n = 0;
      while (!eof() && peek() != '}') {
        const int d = digit(peek());
        if (d < 0 || ++n > 8) syntax("invalid hexadecimal escape");
        v = v * 16 + (uint32_t)d;
        pos_++;
      }
      if (eof() || n == 0) syntax("invalid hexadecimal escape");
      pos_++;
    } else {
      for (int k = 0; k < 2; k++) {
        const int d = digit(peek());
        if (d < 0) syntax("invalid hexadecimal escape");
        v = v * 16 + (uint32_t)d;
        pos_++;
      }
    }
    if (v > MAX_CP || (v >= 0xD800 && v <= 0xDFFF)) syntax("invalid Unicode scalar value");
    return v;
  }

  // after `[`: the class, case-folded and negated as the flags and `^` ask
  Set cls(const Flags& f) {
    const bool neg = peek() == '^';
    if (neg) pos_++;
    Set plain, perl;  // plain items fold under (?i); Perl classes are case-closed already
    bool first = true;
    for (;;) {
      if (eof()) syntax("unclosed character class");
      const char c = peek();
      if (c == ']' && !first) { pos_++; break; }
      if ((c == '&' && peek(1) == '&') || (c == '-' && peek(1) == '-') || (c == '~' && peek(1) == '~'))
        unsupported("class set operation");
      first = false;
      if (c == '[' && peek(1) == ':') {
        const size_t close = p_.find(":]", pos_ + 2);
        if (close != std::string::npos) {
          std::string nm = p_.substr(pos_ + 2, close - pos_ - 2);
          const bool pneg = !nm.empty() && nm[0] == '^';
          if (pneg) nm.erase(0, 1);
          Set s;
          if (!posix(nm, &s)) syntax("invalid ASCII class name");
          if (pneg) s.negate();
          pos_ = close + 2;
          plain.merge(s);
          continue;
        }
      }
      if (c == '[') {
        pos_++;
        Set nested = cls(f);
        if (nested.perl) perl.merge(nested); else plain.r.insert(plain.r.end(), nested.r.begin(), nested.r.end());
        continue;
      }
      uint32_t lo;
      if (c == '\\') {
        pos_++;
        Set s;
        if (escape(&s)) {
          if (peek() == '-' && peek(1) != ']') syntax("invalid range in character class");
          perl.merge(s);
          continue;
        }
        lo = s.r[0].lo;
      } else lo = next_cp();
      uint32_t hi = lo;
      if (peek() == '-' && peek(1) != ']' && peek(1) != '\0') {
        if (peek(1) == '-') unsupported("class set operation");
        pos_++;
        if (peek() == '[') syntax("invalid range in character class");
        if (peek() == '\\') {
          pos_++;
          Set s;
          if (escape(&s)) syntax("invalid range in character class");
          hi = s.r[0].lo;
        } else hi = next_cp();
        if (hi < lo) syntax("invalid range in character class");
      }
      plain.add(lo, hi);
    }
    plain.norm();
    if (f.i) plain.fold();
    plain.merge(perl);
    plain.norm();
    if (neg) plain.negate();
    return plain;
  }
  static bool posix(const std::string& n, Set* s) {
    if (n == "alnum") { s->add('0', '9'); s->add('A', 'Z'); s->add('a', 'z'); }
    else if (n == "alpha") { s->add('A', 'Z'); s->add('a', 'z'); }
    else if (n == "ascii") s->add(0, 0x7F);
    else if (n == "blank") { s->add('\t', '\t'); s->add(' ', ' '); }
    else if (n == "cntrl") { s->add(0, 0x1F); s->add(0x7F, 0x7F); }
    else if (n == "digit") s->add('0', '9');
    else if (n == "graph") s->add('!', '~');
    else if (n == "lower") s->add('a', 'z');
    else if (n == "print") s->add(' ', '~');
    else if (n == "punct") { s->add('!', '/'); s->add(':', '@'); s->add('[', '`'); s->add('{', '~'); }
    else if (n == "space") { s->add('\t', '\r'); s->add(' ', ' '); }
    else if (n == "upper") s->add('A', 'Z');
    else if (n == "word") { s->add('0', '9'); s->add('A', 'Z'); s->add('_', '_'); s->add('a', 'z'); }
    else if (n == "xdigit") { s->add('0', '9'); s->add('A', 'F'); s->add('a', 'f'); }
    else return false;
    s->norm();
    return true;
  }
};

// Thompson NFA: CHAR states consume one code point of `set` and go to next[0]; SPLIT states branch without input
struct State {
  enum Kind { Char, Split, Match } kind;
  uint32_t set = 0;
  std::vector<uint32_t> next;
};

class Regex {
 public:
  explicit Regex(const std::string& pattern) {
    Node root = Parser(pattern).parse();
    states_.push_back({State::Match, 0, {}});
    start_nfa_ = compile(root, 0);
    // DFA state 0: dead (no NFA state, not accepting)
    intern({});
    start_ = intern(closure({start_nfa_}));
  }
  uint32_t num_states() const { return (uint32_t)states_.size(); }
  uint64_t transitions() const { return transitions_; }

  // Ordinals of the terms of field `f` that the pattern matches whole, ascending. The automaton state is kept per
  // code point boundary of the previous term, so each term resumes at its common prefix with the one before; a state
  // that dies at depth d skips, by binary search, every later term that shares those d bytes.
  std::vector<uint32_t> matching_terms(const ImageView& img, uint32_t f) {
    const QwImgField& F = img.fields[f];
    const uint32_t end = F.first_term + F.num_terms;
    std::vector<uint32_t> out;
    std::vector<std::pair<uint32_t, uint32_t>> stack{{0u, start_}};  // (byte depth, automaton state)
    const uint8_t* prev = nullptr;
    uint32_t prev_len = 0;
    auto bytes = [&](uint32_t t) { return img.term_bytes + img.terms[t].bytes_off; };
    for (uint32_t t = F.first_term; t < end;) {
      const uint8_t* b = bytes(t);
      const uint32_t len = img.terms[t].bytes_len;
      uint32_t lcp = 0;
      while (lcp < len && lcp < prev_len && b[lcp] == prev[lcp]) lcp++;
      while (stack.back().first > lcp) stack.pop_back();
      uint32_t d = stack.back().first, s = stack.back().second;
      while (d < len && s != 0) {
        uint32_t n;
        const uint32_t cp = decode(b + d, len - d, &n);
        s = step(s, cp);
        d += n;
        stack.push_back({d, s});
      }
      prev = b;
      prev_len = len;
      if (s == 0) {
        // every term that starts with b[0, d) dies at the same depth
        uint32_t lo = t + 1, hi = end;
        while (lo < hi) {
          const uint32_t mid = lo + (hi - lo) / 2;
          if (img.terms[mid].bytes_len >= d && memcmp(bytes(mid), b, d) == 0) lo = mid + 1; else hi = mid;
        }
        t = lo;
        continue;
      }
      if (accept_[s]) out.push_back(t);
      t++;
    }
    return out;
  }

  // whole-string match of UTF-8 bytes (tests and the walk share step())
  bool matches(const uint8_t* b, uint32_t len) {
    uint32_t s = start_, d = 0;
    while (d < len && s != 0) {
      uint32_t n;
      s = step(s, decode(b + d, len - d, &n));
      d += n;
    }
    return s != 0 && accept_[s];
  }

 private:
  std::vector<State> states_;
  std::vector<Set> sets_;
  uint32_t start_nfa_ = 0, start_ = 0;
  std::map<std::vector<uint32_t>, uint32_t> index_;  // NFA states of each automaton state -> its id
  std::vector<const std::vector<uint32_t>*> dstates_;  // id -> its key in index_ (map keys do not move)
  std::vector<uint8_t> accept_;
  uint64_t stored_ = 0;                                // NFA states held by all keys
  std::unordered_map<uint64_t, uint32_t> trans_;
  uint64_t transitions_ = 0;

  uint32_t add(State s) {
    if (states_.size() >= MAX_STATES)
      fail(QWGPU_EUNSUPPORTED, "regex automaton of more than %u states is not implemented on the GPU path", MAX_STATES);
    states_.push_back(std::move(s));
    return (uint32_t)states_.size() - 1;
  }
  // whether `n` can consume a code point: a repetition at most 0 times, or a concatenation / alternation of nodes that
  // cannot, only ever matches the empty string
  static bool consumes(const Node& n) {
    if (n.kind == Node::Chars) return true;
    if (n.kind == Node::Rep && n.max == 0) return false;
    for (const Node& k : n.kids) if (consumes(k)) return true;
    return false;
  }
  // entry state of `n` whose exit continues at `next`
  uint32_t compile(const Node& n, uint32_t next) {
    switch (n.kind) {
      case Node::Empty: return next;
      case Node::Chars:
        sets_.push_back(n.set);
        return add({State::Char, (uint32_t)sets_.size() - 1, {next}});
      case Node::Cat:
        for (size_t k = n.kids.size(); k-- > 0;) next = compile(n.kids[k], next);
        return next;
      case Node::Alt: {
        if (n.kids.size() == 1) return compile(n.kids[0], next);
        std::vector<uint32_t> outs;
        for (const Node& k : n.kids) outs.push_back(compile(k, next));
        return add({State::Split, 0, outs});
      }
      case Node::Rep: {
        const Node& body = n.kids[0];
        // a body that only matches the empty string adds nothing; every other copy below adds at least one state, so the
        // state bound ends any large count
        if (!consumes(body)) return next;
        uint32_t t = next;
        if (n.max == UINT32_MAX) {
          const uint32_t loop = add({State::Split, 0, {}});
          const uint32_t entry = compile(body, loop);
          states_[loop].next = {entry, next};
          t = loop;
        } else {
          for (uint32_t k = n.min; k < n.max; k++) {
            const uint32_t entry = compile(body, t);
            t = add({State::Split, 0, {entry, next}});
          }
        }
        for (uint32_t k = 0; k < n.min; k++) t = compile(body, t);
        return t;
      }
    }
    return next;
  }
  std::vector<uint32_t> closure(const std::vector<uint32_t>& seeds) {
    std::vector<uint8_t> seen(states_.size(), 0);
    std::vector<uint32_t> stack = seeds, out;
    while (!stack.empty()) {
      const uint32_t s = stack.back();
      stack.pop_back();
      if (seen[s]) continue;
      seen[s] = 1;
      const State& st = states_[s];
      if (st.kind == State::Split) for (uint32_t x : st.next) stack.push_back(x);
      else out.push_back(s);  // Char, or Match (state 0)
    }
    std::sort(out.begin(), out.end());
    return out;
  }
  uint32_t intern(const std::vector<uint32_t>& key) {
    auto it = index_.find(key);
    if (it != index_.end()) return it->second;
    if (dstates_.size() >= MAX_DFA_STATES)
      fail(QWGPU_EUNSUPPORTED, "regex walk of more than %u automaton states is not implemented on the GPU path", MAX_DFA_STATES);
    stored_ += key.size();
    if (stored_ > MAX_DFA_ENTRIES)
      fail(QWGPU_EUNSUPPORTED, "regex walk holding more than %u NFA states in its automaton states is not implemented on the GPU path", MAX_DFA_ENTRIES);
    const uint32_t id = (uint32_t)dstates_.size();
    dstates_.push_back(&index_.emplace(key, id).first->first);
    accept_.push_back(!key.empty() && key[0] == 0);  // NFA state 0 = Match
    return id;
  }
  uint32_t step(uint32_t s, uint32_t cp) {
    transitions_++;
    const uint64_t k = ((uint64_t)s << 22) | cp;
    auto it = trans_.find(k);
    if (it != trans_.end()) return it->second;
    std::vector<uint32_t> seeds;
    bool perl_tested = false;
    for (uint32_t q : *dstates_[s]) {
      const State& st = states_[q];
      if (st.kind != State::Char) continue;
      const Set& set = sets_[st.set];
      perl_tested |= set.perl;
      if (set.has(cp)) seeds.push_back(st.next[0]);
    }
    if (perl_tested && cp >= 0x80)
      fail(QWGPU_EUNSUPPORTED, "regex Perl classes (\\d \\s \\w) tested against non-ASCII terms are not implemented on the GPU path (their definitions are Unicode)");
    const uint32_t to = seeds.empty() ? 0u : intern(closure(seeds));
    trans_.emplace(k, to);
    return to;
  }
  // one code point of a term; a byte that does not start a valid sequence reads as a value no class holds
  static uint32_t decode(const uint8_t* b, uint32_t avail, uint32_t* n) {
    const uint8_t c = b[0];
    const uint32_t len = c < 0x80 ? 1 : (c >> 5) == 6 ? 2 : (c >> 4) == 14 ? 3 : (c >> 3) == 30 ? 4 : 0;
    if (len == 0 || len > avail) { *n = 1; return MAX_CP + 1 + c; }
    uint32_t cp = len == 1 ? c : len == 2 ? (c & 0x1F) : len == 3 ? (c & 0x0F) : (c & 0x07);
    for (uint32_t k = 1; k < len; k++) {
      if ((b[k] & 0xC0) != 0x80) { *n = 1; return MAX_CP + 1 + c; }
      cp = (cp << 6) | (b[k] & 0x3F);
    }
    *n = len;
    return cp;
  }
};

// regex_query.rs regex_has_case_insensitive_flag: a plain string test — the pattern starts with `(?` and the text up
// to the first `)` holds an `i` (so `(?-i)ABC` counts as case-insensitive, and is not prefixed)
inline bool has_case_insensitive_flag(const std::string& re) {
  if (re.compare(0, 2, "(?") != 0) return false;
  const size_t close = re.find(')', 2);
  return close != std::string::npos && re.find('i', 2) < close;
}

}  // namespace rx
}  // namespace qw
