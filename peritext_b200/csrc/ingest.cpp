// ingest.cpp — native wire-format ingest: the reference's `Change[]` JSON (reference src/micromerge.ts:60-71, 143-212;
// mark ops src/peritext.ts:11-65; the shape saved in traces/*.json) -> packed op logs + per-change admission table
// (include/peritext_b200.h).  Host only, multithreaded over logs.  Same packing rules as peritext_b200/packing.py
// (`pack_logs`), which stays as the readable specification and is what tests/test_ingest.py compares against:
//   * opIds "ctr@actor" -> (ctr, rank of the actorId among the log's actors in JS string order = UTF-16 code units,
//     src/micromerge.ts:812-827); strings are kept as UTF-16 so that the order is the reference's
//   * ROOT-map ops are replayed with LWW on the opId to find the text list (src/micromerge.ts:571-603, 446-463)
//   * JSON-saved traces lost their Symbol fields: missing `obj` = ROOT, insert without `elemId` = HEAD (SURVEY.md §9.3 Q6)
//   * link attrs / multi-character values are interned per batch in first-appearance order, comment ids are ranked by JS
//     string order (sortBy, src/peritext.ts:318); counters far beyond the op count are re-ranked densely
//   * every Change also yields one pt_change_rec (actor, seq, deps) for the admission pre-pass (src/micromerge.ts:501-509)
//   * the ops that are not packed (ROOT-map ops, other objects) and each change's startOp are kept as extras (pt_change_extra,
//     packing.change_extras) with each log's list id, so pt_batch_render_changes_json can give the changes back exactly
#include <algorithm>
#include <atomic>
#include <cstdint>
#include <cstring>
#include <map>
#include <string>
#include <thread>
#include <unordered_map>
#include <vector>

#include "../../include/peritext_b200.h"

namespace {

using u16s = std::u16string;

struct JV {
    enum T { Null, Bool, Num, Str, Arr, Obj } t = Null;
    bool b = false;
    std::string num;                 // raw number text
    u16s s;
    std::vector<JV> a;
    std::vector<std::pair<u16s, JV>> o;
    const JV* get(const char16_t* k) const {
        if (t != Obj) return nullptr;
        for (auto& kv : o) if (kv.first == k) return &kv.second;
        return nullptr;
    }
};

struct Parser {
    const unsigned char* p; const unsigned char* e; std::string err;
    void ws() { while (p < e && (*p == ' ' || *p == '\n' || *p == '\r' || *p == '\t')) p++; }
    bool fail(const char* m) { if (err.empty()) err = m; return false; }
    static int hex(unsigned char c) { return c >= '0' && c <= '9' ? c - '0' : c >= 'a' && c <= 'f' ? c - 'a' + 10 : c >= 'A' && c <= 'F' ? c - 'A' + 10 : -1; }
    bool str(u16s& out) {
        if (p >= e || *p != '"') return fail("expected string");
        p++;
        while (p < e && *p != '"') {
            unsigned char c = *p++;
            if (c == '\\') {
                if (p >= e) return fail("bad escape");
                unsigned char d = *p++;
                switch (d) {
                    case '"': out.push_back(u'"'); break; case '\\': out.push_back(u'\\'); break; case '/': out.push_back(u'/'); break;
                    case 'b': out.push_back(8); break; case 'f': out.push_back(12); break; case 'n': out.push_back(10); break;
                    case 'r': out.push_back(13); break; case 't': out.push_back(9); break;
                    case 'u': {
                        if (e - p < 4) return fail("bad \\u escape");
                        int v = 0;
                        for (int k = 0; k < 4; k++) { int h = hex(p[k]); if (h < 0) return fail("bad \\u escape"); v = v * 16 + h; }
                        p += 4; out.push_back((char16_t)v); break;     // surrogates pass through as code units
                    }
                    default: return fail("bad escape");
                }
            } else if (c < 0x80) out.push_back(c);
            else {   // UTF-8 -> UTF-16
                uint32_t cp; int n;
                if ((c & 0xE0) == 0xC0) { cp = c & 0x1F; n = 1; } else if ((c & 0xF0) == 0xE0) { cp = c & 0x0F; n = 2; }
                else if ((c & 0xF8) == 0xF0) { cp = c & 0x07; n = 3; } else return fail("bad UTF-8");
                if (e - p < n) return fail("bad UTF-8");
                for (int k = 0; k < n; k++) { if ((p[k] & 0xC0) != 0x80) return fail("bad UTF-8"); cp = (cp << 6) | (p[k] & 0x3F); }
                p += n;
                if (cp >= 0x10000) { cp -= 0x10000; out.push_back((char16_t)(0xD800 + (cp >> 10))); out.push_back((char16_t)(0xDC00 + (cp & 0x3FF))); }
                else out.push_back((char16_t)cp);
            }
        }
        if (p >= e) return fail("unterminated string");
        p++;
        return true;
    }
    bool value(JV& v, int depth = 0) {
        if (depth > 64) return fail("nesting too deep");
        ws();
        if (p >= e) return fail("unexpected end");
        unsigned char c = *p;
        if (c == '{') {
            v.t = JV::Obj; p++; ws();
            if (p < e && *p == '}') { p++; return true; }
            for (;;) {
                ws(); u16s k; if (!str(k)) return false;
                ws(); if (p >= e || *p != ':') return fail("expected ':'");
                p++;
                v.o.emplace_back(std::move(k), JV());
                if (!value(v.o.back().second, depth + 1)) return false;
                ws(); if (p < e && *p == ',') { p++; continue; }
                if (p < e && *p == '}') { p++; return true; }
                return fail("expected ',' or '}'");
            }
        }
        if (c == '[') {
            v.t = JV::Arr; p++; ws();
            if (p < e && *p == ']') { p++; return true; }
            for (;;) {
                v.a.emplace_back();
                if (!value(v.a.back(), depth + 1)) return false;
                ws(); if (p < e && *p == ',') { p++; continue; }
                if (p < e && *p == ']') { p++; return true; }
                return fail("expected ',' or ']'");
            }
        }
        if (c == '"') { v.t = JV::Str; return str(v.s); }
        if (c == 't' && e - p >= 4 && !memcmp(p, "true", 4)) { v.t = JV::Bool; v.b = true; p += 4; return true; }
        if (c == 'f' && e - p >= 5 && !memcmp(p, "false", 5)) { v.t = JV::Bool; v.b = false; p += 5; return true; }
        if (c == 'n' && e - p >= 4 && !memcmp(p, "null", 4)) { v.t = JV::Null; p += 4; return true; }
        if (c == '-' || (c >= '0' && c <= '9')) {
            const unsigned char* s0 = p;
            while (p < e && (*p == '-' || *p == '+' || *p == '.' || *p == 'e' || *p == 'E' || (*p >= '0' && *p <= '9'))) p++;
            v.t = JV::Num; v.num.assign((const char*)s0, p - s0); return true;
        }
        return fail("unexpected character");
    }
};

// canonical JSON text (python json.dumps(obj, sort_keys=True, separators=(",", ":"), ensure_ascii=False)), as UTF-8
void utf16_to_utf8(const u16s& s, std::string& out) {
    for (size_t i = 0; i < s.size(); i++) {
        uint32_t c = s[i];
        if (c >= 0xD800 && c < 0xDC00 && i + 1 < s.size() && s[i + 1] >= 0xDC00 && s[i + 1] < 0xE000) { c = 0x10000 + ((c - 0xD800) << 10) + (s[i + 1] - 0xDC00); i++; }
        if (c < 0x80) out.push_back((char)c);
        else if (c < 0x800) { out.push_back((char)(0xC0 | (c >> 6))); out.push_back((char)(0x80 | (c & 0x3F))); }
        else if (c < 0x10000) { out.push_back((char)(0xE0 | (c >> 12))); out.push_back((char)(0x80 | ((c >> 6) & 0x3F))); out.push_back((char)(0x80 | (c & 0x3F))); }
        else { out.push_back((char)(0xF0 | (c >> 18))); out.push_back((char)(0x80 | ((c >> 12) & 0x3F))); out.push_back((char)(0x80 | ((c >> 6) & 0x3F))); out.push_back((char)(0x80 | (c & 0x3F))); }
    }
}
void canon_str(const u16s& s, std::string& out) {
    out.push_back('"');
    u16s plain;
    for (char16_t c : s) {
        const char* esc = nullptr; char buf[8];
        switch (c) { case u'"': esc = "\\\""; break; case u'\\': esc = "\\\\"; break; case 10: esc = "\\n"; break; case 13: esc = "\\r"; break;
                     case 9: esc = "\\t"; break; case 8: esc = "\\b"; break; case 12: esc = "\\f"; break; default: break; }
        if (!esc && c < 0x20) { snprintf(buf, sizeof buf, "\\u%04x", (unsigned)c); esc = buf; }
        if (esc) { utf16_to_utf8(plain, out); plain.clear(); out += esc; } else plain.push_back(c);
    }
    utf16_to_utf8(plain, out);
    out.push_back('"');
}
void canon(const JV& v, std::string& out) {
    switch (v.t) {
        case JV::Null: out += "null"; break;
        case JV::Bool: out += v.b ? "true" : "false"; break;
        case JV::Num: out += v.num; break;
        case JV::Str: canon_str(v.s, out); break;
        case JV::Arr: out.push_back('['); for (size_t i = 0; i < v.a.size(); i++) { if (i) out.push_back(','); canon(v.a[i], out); } out.push_back(']'); break;
        case JV::Obj: {
            std::vector<const std::pair<u16s, JV>*> ks; for (auto& kv : v.o) ks.push_back(&kv);
            std::stable_sort(ks.begin(), ks.end(), [](auto a, auto b) { return a->first < b->first; });
            out.push_back('{');
            for (size_t i = 0; i < ks.size(); i++) { if (i) out.push_back(','); canon_str(ks[i]->first, out); out.push_back(':'); canon(ks[i]->second, out); }
            out.push_back('}'); break;
        }
    }
}

bool parse_opid(const u16s& s, uint64_t& ctr, u16s& actor) {       // ^([0-9]+)@(.*)$  (src/micromerge.ts:815)
    size_t i = 0; ctr = 0;
    while (i < s.size() && s[i] >= u'0' && s[i] <= u'9') { ctr = ctr * 10 + (s[i] - u'0'); i++; if (ctr > (1ull << 62)) return false; }
    if (i == 0 || i >= s.size() || s[i] != u'@') return false;
    actor.assign(s, i + 1, u16s::npos);
    return true;
}

struct Bound { uint32_t type = 0; uint64_t ctr = 0; int actor = -1; };
struct InsDel { uint64_t ctr, rctr; int actor, ractor; uint32_t kind, tok; };
struct Mark { uint64_t ctr; int actor; bool add; uint32_t mt; Bound sb, eb; int attr_kind; uint32_t attr_local; uint32_t arrival; };   // attr_kind 0 none, 1 link, 2 comment
struct Change { int actor; uint32_t seq; std::vector<std::pair<int, uint32_t>> deps; uint32_t n_ops; };
struct Extra { uint32_t change, pos; uint64_t start_op; bool none; std::string op; };   // an op off the text list, or startOp alone
struct LogB {
    std::vector<u16s> actors;                       // local actor ids, first-appearance order
    std::unordered_map<std::string, int> actor_ix;  // key: raw bytes of the u16 string
    std::vector<InsDel> insdel; std::vector<Mark> marks; std::vector<Change> changes;
    std::vector<Extra> extras; u16s list_id;
    std::vector<u16s> values; std::unordered_map<std::string, uint32_t> value_ix;          // local pools (merged in log order)
    std::vector<std::string> links; std::unordered_map<std::string, uint32_t> link_ix;
    std::vector<u16s> comments; std::vector<std::string> comment_attrs; std::unordered_map<std::string, uint32_t> comment_ix;
    uint64_t max_ctr = 0;
    std::string err;
    static std::string key(const u16s& s) { return std::string((const char*)s.data(), s.size() * 2); }
    int actor_of(const u16s& a) { auto k = key(a); auto it = actor_ix.find(k); if (it != actor_ix.end()) return it->second; int ix = (int)actors.size(); actors.push_back(a); actor_ix.emplace(std::move(k), ix); return ix; }
};

const char16_t* kMarkTypes[4] = {u"strong", u"em", u"comment", u"link"};
const char16_t* kBoundTypes[4] = {u"before", u"after", u"startOfText", u"endOfText"};

bool build_log(const JV& root, LogB& b) {
    if (root.t != JV::Arr) { b.err = "a log must be a JSON array of Change objects"; return false; }
    // which list does ["text"] resolve to?  LWW over the ROOT-map ops (src/micromerge.ts:571-603)
    std::map<u16s, std::pair<uint64_t, u16s>> key_meta; std::map<u16s, u16s> children;
    for (auto& ch : root.a) {
        const JV* ops = ch.get(u"ops");
        if (!ops || ops->t != JV::Arr) { b.err = "change without ops"; return false; }
        for (auto& op : ops->a) {
            const JV* obj = op.get(u"obj");
            if (obj && !(obj->t == JV::Null || (obj->t == JV::Str && obj->s == u"_root"))) continue;
            const JV* key = op.get(u"key"); const JV* act = op.get(u"action");
            if (!key || key->t != JV::Str || !act || act->t != JV::Str || act->s == u"addMark" || act->s == u"removeMark") continue;
            const JV* id = op.get(u"opId"); uint64_t c; u16s a;
            if (!id || id->t != JV::Str || !parse_opid(id->s, c, a)) { b.err = "Invalid operation ID"; return false; }
            auto it = key_meta.find(key->s);
            if (it == key_meta.end() || it->second < std::make_pair(c, a)) {
                key_meta[key->s] = std::make_pair(c, a);
                if (act->s == u"makeList" || act->s == u"makeMap") children[key->s] = id->s;
            }
        }
    }
    auto lt = children.find(u"text");
    const bool have_list = lt != children.end();
    if (have_list) b.list_id = lt->second;
    for (auto& ch : root.a) {
        Change C; C.n_ops = 0;
        const JV* so = ch.get(u"startOp");
        const bool have_start = so && so->t == JV::Num;
        const uint64_t start_op = have_start ? strtoull(so->num.c_str(), nullptr, 10) : 0;
        const size_t ex0 = b.extras.size();
        uint64_t first_ctr = 0;
        uint32_t op_pos = 0;
        const JV* ca = ch.get(u"actor"); const JV* cs = ch.get(u"seq");
        if (!ca || ca->t != JV::Str || !cs || cs->t != JV::Num) { b.err = "change without actor/seq"; return false; }
        C.actor = b.actor_of(ca->s); C.seq = (uint32_t)strtoull(cs->num.c_str(), nullptr, 10);
        if (const JV* deps = ch.get(u"deps")) if (deps->t == JV::Obj)
            for (auto& kv : deps->o) { if (kv.second.t != JV::Num) { b.err = "bad deps"; return false; } C.deps.emplace_back(b.actor_of(kv.first), (uint32_t)strtoull(kv.second.num.c_str(), nullptr, 10)); }
        const JV* ops = ch.get(u"ops");
        for (auto& op : ops->a) {
            const uint32_t pos = op_pos++;
            const JV* obj = op.get(u"obj");
            if (!have_list || !obj || obj->t != JV::Str || obj->s != lt->second) {
                Extra x{(uint32_t)b.changes.size(), pos, start_op, false, std::string()};
                canon(op, x.op);
                b.extras.push_back(std::move(x));
                continue;
            }
            const JV* id = op.get(u"opId"); const JV* act = op.get(u"action");
            uint64_t ctr; u16s actor;
            if (!id || id->t != JV::Str || !parse_opid(id->s, ctr, actor)) { b.err = "Invalid operation ID"; return false; }
            if (!act || act->t != JV::Str) { b.err = "op without action"; return false; }
            const int ai = b.actor_of(actor);
            b.max_ctr = std::max(b.max_ctr, ctr);
            if (C.n_ops++ == 0) first_ctr = ctr;
            auto elem = [&](const JV* e, uint64_t& c, int& a) -> bool {       // elemId -> (ctr, actor); false: HEAD / absent
                if (!e || e->t != JV::Str || e->s == u"_head") return false;
                u16s ea; if (!parse_opid(e->s, c, ea)) { b.err = "Invalid operation ID"; return false; }
                a = b.actor_of(ea); return true;
            };
            if (act->s == u"addMark" || act->s == u"removeMark") {
                Mark m{}; m.ctr = ctr; m.actor = ai; m.add = act->s == u"addMark"; m.attr_kind = 0; m.attr_local = 0; m.arrival = (uint32_t)b.insdel.size();
                const JV* mt = op.get(u"markType"); m.mt = 4;
                if (mt && mt->t == JV::Str) for (uint32_t k = 0; k < 4; k++) if (mt->s == kMarkTypes[k]) m.mt = k;
                if (m.mt == 4) { b.err = "unknown markType"; return false; }
                for (int side = 0; side < 2; side++) {
                    const JV* bd = op.get(side ? u"end" : u"start"); Bound& B = side ? m.eb : m.sb; B.type = 4;
                    const JV* ty = bd ? bd->get(u"type") : nullptr;
                    if (ty && ty->t == JV::Str) for (uint32_t k = 0; k < 4; k++) if (ty->s == kBoundTypes[k]) B.type = k;
                    if (B.type == 4) { b.err = "bad mark boundary"; return false; }
                    if (B.type <= 1) { if (!elem(bd->get(u"elemId"), B.ctr, B.actor)) { if (b.err.empty()) b.err = "mark boundary without elemId"; return false; } }
                }
                const JV* attrs = op.get(u"attrs");
                if (attrs && attrs->t != JV::Null) {
                    if (m.mt == 3) {
                        std::string k; canon(*attrs, k);
                        auto it = b.link_ix.find(k);
                        if (it == b.link_ix.end()) { it = b.link_ix.emplace(k, (uint32_t)b.links.size()).first; b.links.push_back(k); }
                        m.attr_kind = 1; m.attr_local = it->second;
                    } else if (m.mt == 2) {
                        const JV* cid = attrs->get(u"id");
                        if (!cid || cid->t != JV::Str) { b.err = "comment mark without attrs.id"; return false; }
                        auto k = LogB::key(cid->s); auto it = b.comment_ix.find(k);
                        if (it == b.comment_ix.end()) { it = b.comment_ix.emplace(k, (uint32_t)b.comments.size()).first; b.comments.push_back(cid->s); std::string ca2; canon(*attrs, ca2); b.comment_attrs.push_back(ca2); }
                        m.attr_kind = 2; m.attr_local = it->second;
                    } else {
                        std::string k; canon(*attrs, k);
                        if (k != "{\"active\":true}") { b.err = "strong/em marks with custom attrs"; return false; }
                    }
                } else if (m.mt == 2) { b.err = "comment mark without attrs"; return false; }
                b.marks.push_back(m);
            } else if (act->s == u"set" && op.get(u"insert") && op.get(u"insert")->t == JV::Bool && op.get(u"insert")->b) {
                InsDel r{}; r.ctr = ctr; r.actor = ai; r.kind = PT_KIND_INSERT; r.rctr = 0; r.ractor = -1;
                if (!elem(op.get(u"elemId"), r.rctr, r.ractor) && !b.err.empty()) return false;
                const JV* v = op.get(u"value");
                if (!v || v->t != JV::Str) { b.err = "Expected value inserted into text to be a string"; return false; }   // src/micromerge.ts:654-656
                const u16s& s = v->s;
                const bool pair = s.size() == 2 && s[0] >= 0xD800 && s[0] < 0xDC00 && s[1] >= 0xDC00 && s[1] < 0xE000;
                if (s.size() == 1) r.tok = s[0];
                else if (pair) r.tok = 0x10000u + ((uint32_t)(s[0] - 0xD800) << 10) + (s[1] - 0xDC00);
                else {
                    auto k = LogB::key(s); auto it = b.value_ix.find(k);
                    if (it == b.value_ix.end()) { it = b.value_ix.emplace(k, (uint32_t)b.values.size()).first; b.values.push_back(s); }
                    r.tok = PT_TOKEN_POOLED | it->second;           // local index, re-mapped at the merge
                }
                b.insdel.push_back(r);
            } else if (act->s == u"del" && (!op.get(u"key") || op.get(u"key")->t == JV::Null)) {
                InsDel r{}; r.ctr = ctr; r.actor = ai; r.kind = PT_KIND_DELETE; r.tok = 0;
                if (!elem(op.get(u"elemId"), r.rctr, r.ractor)) { if (b.err.empty()) b.err = "List element not found: _head"; return false; }
                b.insdel.push_back(r);
            } else { b.err = "unsupported action on a list"; return false; }               // src/micromerge.ts:567
        }
        // a change whose ops cannot say its startOp keeps it in an entry without an op
        if (b.extras.size() == ex0 && have_start && (C.n_ops == 0 || first_ctr != start_op))
            b.extras.push_back(Extra{(uint32_t)b.changes.size(), 0, start_op, true, std::string()});
        b.changes.push_back(std::move(C));
    }
    return true;
}

}  // namespace

struct pt_ingest {
    std::string err;
    std::vector<pt_log_desc> desc; std::vector<pt_insdel_rec> insdel; std::vector<pt_mark_rec> marks;
    std::vector<pt_change_desc> cdesc; std::vector<pt_change_rec> changes; std::vector<pt_dep_rec> deps;
    // pools: concatenated bytes + offsets
    struct Pool { std::vector<uint8_t> data; std::vector<uint64_t> off{0}; void add(const void* p, size_t n) { data.insert(data.end(), (const uint8_t*)p, (const uint8_t*)p + n); off.push_back(data.size()); } void clear() { data.clear(); off.assign(1, 0); } };
    Pool values, links, comments, comment_attrs, actors, counters;   // actors / counters: per log ranges via *_first
    Pool list_ids, extra_ops;                                        // one entry per log; one per extra with an op
    std::vector<pt_change_extra> extras;
    std::vector<uint64_t> actors_first{0}, counters_first{0};
};

extern "C" {

int pt_ingest_create(pt_ingest** out) { if (!out) return PT_ERR_INVALID; *out = new pt_ingest(); return PT_OK; }
void pt_ingest_destroy(pt_ingest* g) { delete g; }
const char* pt_ingest_error(pt_ingest* g) { return g ? g->err.c_str() : "null handle"; }

int pt_ingest_parse(pt_ingest* g, const char* const* logs_json, const uint64_t* lens, uint32_t n_logs, int threads) {
    if (!g || (n_logs && (!logs_json || !lens))) return PT_ERR_INVALID;
    g->err.clear();
    std::vector<LogB> B(n_logs);
    {
        std::atomic<uint32_t> next{0};
        int T = threads > 0 ? threads : (int)std::max(1u, std::thread::hardware_concurrency());
        T = (int)std::min<uint32_t>((uint32_t)T, std::max(1u, n_logs));
        auto work = [&]() {
            for (;;) {
                const uint32_t i = next.fetch_add(1);
                if (i >= n_logs) break;
                Parser P{(const unsigned char*)logs_json[i], (const unsigned char*)logs_json[i] + lens[i], {}};
                JV root;
                if (!P.value(root)) { B[i].err = "JSON: " + P.err; continue; }
                P.ws();
                if (P.p != P.e) { B[i].err = "JSON: trailing characters"; continue; }
                build_log(root, B[i]);
            }
        };
        std::vector<std::thread> th;
        for (int t = 1; t < T; t++) th.emplace_back(work);
        work();
        for (auto& t : th) t.join();
    }
    for (uint32_t i = 0; i < n_logs; i++) if (!B[i].err.empty()) { g->err = "log " + std::to_string(i) + ": " + B[i].err; return PT_ERR_INVALID; }
    // merge the local pools in log order (first-appearance order over the whole batch, as the sequential packer does)
    g->values.clear(); g->links.clear(); g->comments.clear(); g->comment_attrs.clear(); g->actors.clear(); g->counters.clear();
    g->list_ids.clear(); g->extra_ops.clear(); g->extras.clear();
    g->actors_first.assign(1, 0); g->counters_first.assign(1, 0);
    std::unordered_map<std::string, uint32_t> vix, lix; std::map<u16s, uint32_t> cset; std::vector<std::string> cattr_of;
    std::vector<std::vector<uint32_t>> vmap(n_logs), lmap(n_logs);
    std::vector<u16s> call; std::vector<std::string> callattr;
    for (uint32_t i = 0; i < n_logs; i++) {
        for (auto& v : B[i].values) { auto k = LogB::key(v); auto it = vix.find(k); if (it == vix.end()) { it = vix.emplace(k, (uint32_t)vix.size()).first; g->values.add(v.data(), v.size() * 2); } vmap[i].push_back(it->second); }
        for (auto& l : B[i].links) { auto it = lix.find(l); if (it == lix.end()) { it = lix.emplace(l, (uint32_t)lix.size()).first; g->links.add(l.data(), l.size()); } lmap[i].push_back(it->second); }
        for (size_t k = 0; k < B[i].comments.size(); k++) if (!cset.count(B[i].comments[k])) { cset.emplace(B[i].comments[k], 0); call.push_back(B[i].comments[k]); callattr.push_back(B[i].comment_attrs[k]); }
    }
    {   // comment ranks: JS string order of the id (UTF-16 code units)
        std::vector<uint32_t> ord(call.size()); for (uint32_t k = 0; k < ord.size(); k++) ord[k] = k;
        std::sort(ord.begin(), ord.end(), [&](uint32_t a, uint32_t b) { return call[a] < call[b]; });
        for (uint32_t r = 0; r < ord.size(); r++) { cset[call[ord[r]]] = r; g->comments.add(call[ord[r]].data(), call[ord[r]].size() * 2); g->comment_attrs.add(callattr[ord[r]].data(), callattr[ord[r]].size()); }
    }
    g->desc.assign(n_logs, pt_log_desc{}); g->cdesc.assign(n_logs, pt_change_desc{});
    uint64_t io = 0, mo = 0, co = 0, dpo = 0;
    for (uint32_t i = 0; i < n_logs; i++) { io += B[i].insdel.size(); mo += B[i].marks.size(); co += B[i].changes.size(); for (auto& c : B[i].changes) dpo += c.deps.size(); }
    g->insdel.assign(io, pt_insdel_rec{}); g->marks.assign(mo, pt_mark_rec{}); g->changes.assign(co, pt_change_rec{}); g->deps.assign(dpo, pt_dep_rec{});
    io = mo = co = dpo = 0;
    for (uint32_t i = 0; i < n_logs; i++) {
        LogB& b = B[i];
        // actor ranks: JS string order
        std::vector<uint32_t> ord(b.actors.size()); for (uint32_t k = 0; k < ord.size(); k++) ord[k] = k;
        std::sort(ord.begin(), ord.end(), [&](uint32_t x, uint32_t y) { return b.actors[x] < b.actors[y]; });
        std::vector<uint32_t> rank(b.actors.size());
        for (uint32_t r = 0; r < ord.size(); r++) { rank[ord[r]] = r; g->actors.add(b.actors[ord[r]].data(), b.actors[ord[r]].size() * 2); }
        g->actors_first.push_back(g->actors.off.size() - 1);
        if (b.actors.size() > 0xFFFF) { g->err = "more than 65535 actors in one log"; return PT_ERR_INVALID; }
        // sparse counters are re-ranked densely (only the ORDER of counters matters to compareOpIds)
        std::map<uint64_t, uint32_t> dense; bool use_dense = false;
        if (b.max_ctr > 2ull * (b.insdel.size() + b.marks.size()) + 16) {
            use_dense = true;
            for (auto& r : b.insdel) { dense[r.ctr]; if (r.rctr) dense[r.rctr]; }
            for (auto& m : b.marks) { dense[m.ctr]; if (m.sb.ctr) dense[m.sb.ctr]; if (m.eb.ctr) dense[m.eb.ctr]; }
            uint32_t k = 1; uint64_t zero = 0; g->counters.add(&zero, 8);
            for (auto& kv : dense) { kv.second = k++; g->counters.add(&kv.first, 8); }
        }
        g->counters_first.push_back(g->counters.off.size() - 1);
        auto dc = [&](uint64_t c) -> uint32_t { return c == 0 ? 0u : use_dense ? dense[c] : (uint32_t)c; };
        if (!use_dense && b.max_ctr > 0x7FFFFFFFull) { g->err = "counter too large"; return PT_ERR_INVALID; }
        pt_log_desc& D = g->desc[i];
        D.insdel_off = io; D.mark_off = mo; D.n_insdel = (uint32_t)b.insdel.size(); D.n_mark = (uint32_t)b.marks.size();
        D.n_actors = (uint32_t)std::max<size_t>(1, b.actors.size()); D.max_ctr = use_dense ? dense[b.max_ctr] : (uint32_t)b.max_ctr;
        for (auto& r : b.insdel) {
            pt_insdel_rec& o = g->insdel[io++];
            o.ctr = dc(r.ctr); o.ref_ctr = dc(r.rctr); o.actor = (uint16_t)rank[r.actor]; o.ref_actor = r.ractor >= 0 ? (uint16_t)rank[r.ractor] : 0;
            uint32_t tok = r.tok;
            if (r.kind == PT_KIND_INSERT && (tok & PT_TOKEN_POOLED)) tok = PT_TOKEN_POOLED | vmap[i][tok & (PT_TOKEN_POOLED - 1)];
            o.payload = (r.kind << 30) | tok;
        }
        for (auto& m : b.marks) {
            pt_mark_rec& o = g->marks[mo++];
            o.ctr = dc(m.ctr); o.actor = (uint16_t)rank[m.actor]; o.kind = (uint8_t)((m.add ? 0 : 1) | (m.mt << 1)); o.bounds = (uint8_t)(m.sb.type | (m.eb.type << 2));
            o.start_ctr = dc(m.sb.ctr); o.end_ctr = dc(m.eb.ctr);
            o.start_actor = m.sb.actor >= 0 ? (uint16_t)rank[m.sb.actor] : 0; o.end_actor = m.eb.actor >= 0 ? (uint16_t)rank[m.eb.actor] : 0;
            o.attr = m.attr_kind == 1 ? lmap[i][m.attr_local] : m.attr_kind == 2 ? cset[b.comments[m.attr_local]] : PT_ATTR_NONE;
            o.arrival = m.arrival; o.reserved = 0;
        }
        pt_change_desc& CD = g->cdesc[i];
        CD.change_off = co; CD.dep_off = dpo; CD.n_changes = (uint32_t)b.changes.size(); CD.n_deps = 0;
        for (auto& c : b.changes) {
            pt_change_rec& o = g->changes[co++];
            o.seq = c.seq; o.actor = (uint16_t)rank[c.actor]; o.n_deps = (uint16_t)c.deps.size(); o.dep_off = CD.n_deps; o.n_ops = c.n_ops;
            for (auto& d : c.deps) { pt_dep_rec& q = g->deps[dpo++]; q.seq = d.second; q.actor = (uint16_t)rank[d.first]; q.reserved = 0; CD.n_deps++; }
        }
        g->list_ids.add(b.list_id.data(), b.list_id.size() * 2);
        for (auto& x : b.extras) {
            uint64_t op = PT_EXTRA_NONE;
            if (!x.none) { op = g->extra_ops.off.size() - 1; g->extra_ops.add(x.op.data(), x.op.size()); }
            g->extras.push_back(pt_change_extra{i, x.change, x.pos, 0, x.start_op, op});
        }
    }
    return PT_OK;
}

int pt_ingest_packed(pt_ingest* g, pt_packed_ops* ops, pt_change_table* ch) {
    if (!g) return PT_ERR_INVALID;
    if (ops) { ops->n_logs = (uint32_t)g->desc.size(); ops->logs = g->desc.data(); ops->insdel = g->insdel.data(); ops->n_insdel_total = g->insdel.size(); ops->marks = g->marks.data(); ops->n_mark_total = g->marks.size(); }
    if (ch) { ch->n_logs = (uint32_t)g->cdesc.size(); ch->logs = g->cdesc.data(); ch->changes = g->changes.data(); ch->n_changes_total = g->changes.size(); ch->deps = g->deps.data(); ch->n_deps_total = g->deps.size(); }
    return PT_OK;
}

int pt_ingest_pool(pt_ingest* g, int kind, const uint8_t** data, const uint64_t** offsets, uint64_t* count, const uint64_t** per_log_first) {
    if (!g || !data || !offsets || !count) return PT_ERR_INVALID;
    pt_ingest::Pool* p = kind == PT_POOL_VALUES ? &g->values : kind == PT_POOL_LINK_ATTRS ? &g->links : kind == PT_POOL_COMMENT_IDS ? &g->comments
                       : kind == PT_POOL_COMMENT_ATTRS ? &g->comment_attrs : kind == PT_POOL_ACTORS ? &g->actors : kind == PT_POOL_COUNTERS ? &g->counters
                       : kind == PT_POOL_LIST_IDS ? &g->list_ids : kind == PT_POOL_EXTRA_OPS ? &g->extra_ops : nullptr;
    if (!p) return PT_ERR_INVALID;
    *data = p->data.data(); *offsets = p->off.data(); *count = p->off.size() - 1;
    if (per_log_first) *per_log_first = kind == PT_POOL_ACTORS ? g->actors_first.data() : kind == PT_POOL_COUNTERS ? g->counters_first.data() : nullptr;
    return PT_OK;
}

int pt_ingest_change_extras(pt_ingest* g, const pt_change_extra** out, uint64_t* n) {
    if (!g || !out || !n) return PT_ERR_INVALID;
    *out = g->extras.data(); *n = g->extras.size();
    return PT_OK;
}

}  // extern "C"
