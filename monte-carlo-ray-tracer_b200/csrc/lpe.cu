// Light path expression compiler (host only): parser, Thompson NFA, subset-construction DFA of the union, dead-state
// collapse. The device side (FILM_MODE_LPE in integrator.cuh) only walks the table this produces.
#include "lpe.h"
#include "mcrt_abi.h"

#include <algorithm>
#include <bitset>
#include <cstring>
#include <map>
#include <stdexcept>

namespace mcrt
{
    namespace
    {
        // The NFA alphabet: the device's symbols, and the camera event C, which starts every string and never comes
        // again, so it has no column in the device table
        constexpr uint32_t SYM_C = 127;
        typedef std::bitset<128> SymSet;

        constexpr uint32_t MAX_REPEAT = 1000;        // {n,m} bounds
        constexpr uint32_t MAX_NESTING = 256;        // parentheses
        constexpr size_t MAX_NFA_STATES = 1u << 16;
        constexpr size_t MAX_DFA_STATES = 16384;     // before the dead states collapse
        // NFA states visited by the subset construction (moves and closures): bounds its host time to well under a
        // second whatever the expressions, since the state limits alone allow ~10^13 steps
        constexpr uint64_t MAX_SUBSET_WORK = 1ull << 27;

        // Events named by the expressions, before the labels are numbered: vertex events, B, C, any light, labels
        struct Atoms
        {
            enum : uint32_t { RD = 1u << 0, RS = 1u << 1, RG = 1u << 2, TS = 1u << 3, TG = 1u << 4, B = 1u << 5, C = 1u << 6,
                              L = 1u << 7, ANY = 0xFFu };
            uint32_t mask = 0;
            std::vector<uint32_t> labels;
        };

        struct Node
        {
            enum Kind { SET, CAT, ALT, REP, EMPTY } kind;
            std::vector<int> kids;
            uint32_t lo = 0, hi = 0;   // REP; hi == UINT32_MAX: unbounded
            Atoms atoms;               // SET
            bool negated = false;      // SET
        };

        struct ParseError { size_t offset; std::string what; };

        // Recursive descent over the expression with whitespace removed (each character keeps its offset)
        struct Parser
        {
            std::vector<char> c;
            std::vector<size_t> at;
            size_t end_offset = 0, pos = 0;
            uint32_t depth = 0;
            std::vector<Node>& nodes;

            Parser(const char* s, std::vector<Node>& n) : nodes(n)
            {
                const size_t len = std::strlen(s);
                for (size_t i = 0; i < len; i++)
                    if (s[i] != ' ' && s[i] != '\t' && s[i] != '\n' && s[i] != '\r') { c.push_back(s[i]); at.push_back(i); }
                end_offset = len;
            }
            bool done() const { return pos >= c.size(); }
            char peek() const { return done() ? '\0' : c[pos]; }
            size_t offset() const { return done() ? end_offset : at[pos]; }
            [[noreturn]] void fail(const std::string& what) const { throw ParseError{ offset(), what }; }
            void expect(char ch)
            {
                if (peek() != ch) fail(done() ? std::string("expected '") + ch + "' before the end" : std::string("expected '") + ch + "', found '" + peek() + "'");
                pos++;
            }
            int add(Node n) { nodes.push_back(std::move(n)); return (int)nodes.size() - 1; }

            uint32_t number()
            {
                if (peek() < '0' || peek() > '9') fail("expected a number");
                uint64_t v = 0;
                while (peek() >= '0' && peek() <= '9')
                {
                    v = v * 10 + (uint64_t)(peek() - '0');
                    if (v > MAX_REPEAT) fail("count above " + std::to_string(MAX_REPEAT));
                    pos++;
                }
                return (uint32_t)v;
            }

            // one event (outside or inside a set)
            void event(Atoms& a)
            {
                const char ch = peek();
                switch (ch)
                {
                    case 'C': pos++; a.mask |= Atoms::C; return;
                    case 'B': pos++; a.mask |= Atoms::B; return;
                    case '.': pos++; a.mask |= Atoms::ANY; return;
                    case 'D': pos++; a.mask |= Atoms::RD; return;
                    case 'G': pos++; a.mask |= Atoms::RG | Atoms::TG; return;
                    case 'S': pos++; a.mask |= Atoms::RS | Atoms::TS; return;
                    case 'R': pos++; a.mask |= Atoms::RD | Atoms::RS | Atoms::RG; return;
                    case 'T': pos++; a.mask |= Atoms::TS | Atoms::TG; return;
                    case 'L':
                    {
                        pos++;
                        if (peek() != '\'') { a.mask |= Atoms::L; return; }
                        pos++;
                        if (peek() < '0' || peek() > '9') fail("a label is a light group index");
                        uint64_t g = 0;
                        while (peek() >= '0' && peek() <= '9')
                        {
                            g = g * 10 + (uint64_t)(peek() - '0');
                            if (g > 0xFFFFFFFEull) fail("label out of range");
                            pos++;
                        }
                        expect('\'');
                        a.labels.push_back((uint32_t)g);
                        return;
                    }
                    case '<':
                    {
                        pos++;
                        const char x = peek();
                        if (x != 'R' && x != 'T' && x != '.') fail(done() ? "unterminated '<'" : std::string("scattering direction must be R, T or ., found '") + x + "'");
                        pos++;
                        const char y = peek();
                        if (y != 'D' && y != 'G' && y != 'S' && y != '.') fail(done() ? "unterminated '<'" : std::string("scattering kind must be D, G, S or ., found '") + y + "'");
                        pos++;
                        expect('>');
                        const uint32_t xr = x != 'T' ? (Atoms::RD | Atoms::RS | Atoms::RG) : 0u, xt = x != 'R' ? (Atoms::TS | Atoms::TG) : 0u;
                        const uint32_t yk = y == '.' ? 0x1Fu : (y == 'D' ? Atoms::RD : (y == 'G' ? (Atoms::RG | Atoms::TG) : (Atoms::RS | Atoms::TS)));
                        a.mask |= (xr | xt) & yk;   // <TD> names no event: the reference's diffuse lobe only reflects
                        return;
                    }
                    default:
                        if (done()) fail("expected an event before the end");
                        fail(std::string("unexpected '") + ch + "'");
                }
            }

            int atom()
            {
                if (peek() == '(')
                {
                    pos++;
                    if (++depth > MAX_NESTING) fail("parentheses nested deeper than " + std::to_string(MAX_NESTING));
                    const int n = alt();
                    expect(')');
                    depth--;
                    return n;
                }
                Node n; n.kind = Node::SET;
                if (peek() == '[')
                {
                    pos++;
                    if (peek() == '^') { n.negated = true; pos++; }
                    if (peek() == ']') fail("empty set");
                    while (peek() != ']')
                    {
                        if (done()) fail("unterminated '['");
                        event(n.atoms);
                    }
                    pos++;
                    return add(std::move(n));
                }
                event(n.atoms);
                return add(std::move(n));
            }

            int repeat()
            {
                int a = atom();
                for (;;)
                {
                    const char ch = peek();
                    Node r; r.kind = Node::REP;
                    if (ch == '*') { pos++; r.lo = 0; r.hi = UINT32_MAX; }
                    else if (ch == '+') { pos++; r.lo = 1; r.hi = UINT32_MAX; }
                    else if (ch == '?') { pos++; r.lo = 0; r.hi = 1; }
                    else if (ch == '{')
                    {
                        pos++;
                        r.lo = number();
                        r.hi = r.lo;
                        if (peek() == ',')
                        {
                            pos++;
                            r.hi = peek() == '}' ? UINT32_MAX : number();
                            if (r.hi < r.lo) fail("{n,m} with m < n");
                        }
                        expect('}');
                    }
                    else return a;
                    r.kids.push_back(a);
                    a = add(std::move(r));
                }
            }

            int cat()
            {
                Node n; n.kind = Node::CAT;
                while (!done() && peek() != '|' && peek() != ')') n.kids.push_back(repeat());
                if (n.kids.empty()) n.kind = Node::EMPTY;
                return add(std::move(n));
            }

            int alt()
            {
                Node n; n.kind = Node::ALT;
                n.kids.push_back(cat());
                while (peek() == '|') { pos++; n.kids.push_back(cat()); }
                if (n.kids.size() == 1) return n.kids[0];
                return add(std::move(n));
            }

            int parse()
            {
                if (c.empty()) fail("empty expression");
                const int n = alt();
                if (!done()) fail(std::string("unexpected '") + peek() + "'");
                return n;
            }
        };

        struct Nfa
        {
            std::vector<std::vector<int>> eps;
            std::vector<int> out;         // symbol edge target, -1 none
            std::vector<SymSet> on;       // its symbols
            std::vector<uint32_t> accept;
            std::vector<SymSet> leaf_sets;   // SET node -> symbols (indexed by node)

            int state()
            {
                if (eps.size() >= MAX_NFA_STATES) throw std::length_error("nfa");
                eps.emplace_back(); out.push_back(-1); on.emplace_back(); accept.push_back(0);
                return (int)eps.size() - 1;
            }
            std::pair<int, int> build(const std::vector<Node>& nodes, int id)
            {
                const Node& n = nodes[id];
                switch (n.kind)
                {
                    case Node::SET:
                    {
                        const int s = state(), e = state();
                        out[s] = e; on[s] = leaf_sets[id];
                        return { s, e };
                    }
                    case Node::EMPTY:
                    {
                        const int s = state(), e = state();
                        eps[s].push_back(e);
                        return { s, e };
                    }
                    case Node::CAT:
                    {
                        std::pair<int, int> f = build(nodes, n.kids[0]);
                        const int s = f.first;
                        int cur = f.second;
                        for (size_t k = 1; k < n.kids.size(); k++)
                        {
                            f = build(nodes, n.kids[k]);
                            eps[cur].push_back(f.first);
                            cur = f.second;
                        }
                        return { s, cur };
                    }
                    case Node::ALT:
                    {
                        const int s = state(), e = state();
                        for (int k : n.kids)
                        {
                            const std::pair<int, int> f = build(nodes, k);
                            eps[s].push_back(f.first);
                            eps[f.second].push_back(e);
                        }
                        return { s, e };
                    }
                    case Node::REP:
                    default:
                    {
                        const int s = state();
                        int cur = s;
                        for (uint32_t k = 0; k < n.lo; k++)
                        {
                            const std::pair<int, int> f = build(nodes, n.kids[0]);
                            eps[cur].push_back(f.first);
                            cur = f.second;
                        }
                        if (n.hi == UINT32_MAX)
                        {
                            const std::pair<int, int> f = build(nodes, n.kids[0]);
                            const int x = state();
                            eps[cur].push_back(x);
                            eps[x].push_back(f.first);
                            eps[f.second].push_back(x);
                            cur = x;
                        }
                        else
                        {
                            for (uint32_t k = n.lo; k < n.hi; k++)
                            {
                                const std::pair<int, int> f = build(nodes, n.kids[0]);
                                const int j = state();
                                eps[cur].push_back(f.first);
                                eps[cur].push_back(j);
                                eps[f.second].push_back(j);
                                cur = j;
                            }
                        }
                        return { s, cur };
                    }
                }
            }
            // epsilon closure of set (sorted, unique)
            void close(std::vector<int>& set, std::vector<uint8_t>& mark) const
            {
                std::vector<int> stack(set);
                for (int q : set) mark[q] = 1;
                while (!stack.empty())
                {
                    const int q = stack.back();
                    stack.pop_back();
                    for (int r : eps[q])
                        if (!mark[r]) { mark[r] = 1; set.push_back(r); stack.push_back(r); }
                }
                for (int q : set) mark[q] = 0;
                std::sort(set.begin(), set.end());
            }
        };

        std::string quoted(const char* s) { return std::string("\"") + s + "\""; }
    }

    // The photon side of the table (lpe.h): the DFA of the reversed expressions, read in emission order, and the join of
    // its states with the forward table's. Fills out.rev_* / join / join_any; returns "" or why the photon mapper must
    // refuse the table (the forward table stays valid for the path tracer).
    static std::string compileReverse(const Nfa& nfa, const std::vector<std::pair<int, int>>& ends, uint32_t n_symbols,
                                      LpeTable& out)
    {
        const size_t nq = nfa.eps.size();
        std::vector<std::vector<int>> reps(nq), rin(nq);   // reversed epsilon and symbol edges
        for (size_t q = 0; q < nq; q++)
        {
            for (int r : nfa.eps[q]) reps[r].push_back((int)q);
            if (nfa.out[q] >= 0) rin[nfa.out[q]].push_back((int)q);
        }
        std::vector<uint32_t> first_of(nq, 0);   // reversed, an expression accepts at its own start
        for (size_t i = 0; i < ends.size(); i++) first_of[ends[i].first] |= 1u << i;

        // subset construction over the device symbols and C (column n_symbols), from the expressions' accepting states
        const uint32_t cols = n_symbols + 1;
        std::map<std::vector<int>, uint32_t> index;
        std::vector<std::vector<int>> sets;
        std::vector<uint32_t> dfa_next, dfa_accept;
        std::vector<uint8_t> mark(nq, 0);
        uint64_t steps = 0;
        auto intern = [&](std::vector<int>& set) -> uint32_t
        {
            std::vector<int> stack(set);
            for (int q : set) mark[q] = 1;
            while (!stack.empty())
            {
                const int q = stack.back();
                stack.pop_back();
                for (int r : reps[q])
                    if (!mark[r]) { mark[r] = 1; set.push_back(r); stack.push_back(r); }
            }
            for (int q : set) mark[q] = 0;
            std::sort(set.begin(), set.end());
            steps += set.size();
            auto it = index.find(set);
            if (it != index.end()) return it->second;
            const uint32_t id = (uint32_t)sets.size();
            uint32_t acc = 0;
            for (int q : set) acc |= first_of[q];
            index.emplace(set, id);
            sets.push_back(set);
            dfa_accept.push_back(acc);
            dfa_next.resize(dfa_next.size() + cols, 0);
            return id;
        };
        {
            std::vector<int> s0;
            for (const auto& e : ends) s0.push_back(e.second);
            std::sort(s0.begin(), s0.end());
            s0.erase(std::unique(s0.begin(), s0.end()), s0.end());
            intern(s0);
        }
        for (uint32_t d = 0; d < sets.size(); d++)
        {
            if (sets.size() > MAX_DFA_STATES)
                return "the reversed expressions need more than " + std::to_string(MAX_DFA_STATES) + " automaton states";
            for (uint32_t col = 0; col < cols; col++)
            {
                steps += sets[d].size();
                if (steps > MAX_SUBSET_WORK)
                    return "the reversed expressions' automaton is too large to build (more than " + std::to_string(MAX_SUBSET_WORK) +
                           " subset-construction steps)";
                const uint32_t sym = col < n_symbols ? col : SYM_C;
                std::vector<int> moved;
                for (int q : sets[d])
                    for (int p : rin[q])
                        if (nfa.on[p].test(sym)) moved.push_back(p);
                std::sort(moved.begin(), moved.end());
                moved.erase(std::unique(moved.begin(), moved.end()), moved.end());
                const uint32_t t = intern(moved);
                dfa_next[(size_t)d * cols + col] = t;
            }
        }

        // A string's C comes first and only once, so a photon history is complete once C is read after it: a state's
        // mask is the accept mask after C. Live: a state from which device symbols lead to a nonzero mask.
        const uint32_t nd = (uint32_t)sets.size();
        std::vector<uint32_t> mask_c(nd);
        for (uint32_t d = 0; d < nd; d++) mask_c[d] = dfa_accept[dfa_next[(size_t)d * cols + n_symbols]];
        std::vector<std::vector<uint32_t>> pred(nd);
        for (uint32_t d = 0; d < nd; d++)
            for (uint32_t col = 0; col < n_symbols; col++) pred[dfa_next[(size_t)d * cols + col]].push_back(d);
        std::vector<uint8_t> live(nd, 0);
        std::vector<uint32_t> work;
        for (uint32_t d = 0; d < nd; d++) if (mask_c[d]) { live[d] = 1; work.push_back(d); }
        while (!work.empty())
        {
            const uint32_t d = work.back();
            work.pop_back();
            for (uint32_t p : pred[d]) if (!live[p]) { live[p] = 1; work.push_back(p); }
        }

        // Moore's refinement of the live states, by mask after C and device-symbol transitions
        std::vector<uint32_t> cls(nd, UINT32_MAX);
        size_t n_cls = 0;
        {
            std::map<uint32_t, uint32_t> by_mask;
            for (uint32_t d = 0; d < nd; d++)
                if (live[d]) cls[d] = by_mask.emplace(mask_c[d], (uint32_t)by_mask.size()).first->second;
            n_cls = by_mask.size();
            std::vector<uint32_t> sig(n_symbols + 1);
            for (;;)
            {
                std::map<std::vector<uint32_t>, uint32_t> by_sig;
                std::vector<uint32_t> refined(nd, UINT32_MAX);
                for (uint32_t d = 0; d < nd; d++)
                {
                    if (!live[d]) continue;
                    sig[0] = cls[d];
                    for (uint32_t col = 0; col < n_symbols; col++) sig[col + 1] = cls[dfa_next[(size_t)d * cols + col]];
                    refined[d] = by_sig.emplace(sig, (uint32_t)by_sig.size()).first->second;
                }
                const bool stable = by_sig.size() == n_cls;
                cls.swap(refined);
                n_cls = by_sig.size();
                if (stable) break;
            }
        }

        // breadth-first numbering from the start (no photon event read yet); each class keeps the shortest history
        // that reaches it, as its parent class and last symbol
        std::vector<uint32_t> number(n_cls, MCRT_LPE_DEAD), order, parent, via;
        if (live[0]) { number[cls[0]] = 0; order.push_back(0); parent.push_back(MCRT_LPE_DEAD); via.push_back(0); }
        for (size_t k = 0; k < order.size(); k++)
            for (uint32_t col = 0; col < n_symbols; col++)
            {
                const uint32_t t = dfa_next[(size_t)order[k] * cols + col];
                if (!live[t] || number[cls[t]] != MCRT_LPE_DEAD) continue;
                if (order.size() >= MCRT_LPE_MAX_STATES)
                    return "the reversed expressions need more than " + std::to_string(MCRT_LPE_MAX_STATES) +
                           " live automaton states (a photon's state keeps 8 bits)";
                number[cls[t]] = (uint32_t)order.size();
                order.push_back(t);
                parent.push_back((uint32_t)k);
                via.push_back(col);
            }

        out.rev_n_states = order.empty() ? 1u : (uint32_t)order.size();
        out.rev_start = order.empty() ? (uint32_t)MCRT_LPE_DEAD : 0u;
        out.rev_next.assign((size_t)out.rev_n_states * n_symbols, (uint8_t)MCRT_LPE_DEAD);
        for (uint32_t k = 0; k < order.size(); k++)
            for (uint32_t col = 0; col < n_symbols; col++)
            {
                const uint32_t t = dfa_next[(size_t)order[k] * cols + col];
                out.rev_next[(size_t)k * n_symbols + col] = (uint8_t)(live[t] ? number[cls[t]] : MCRT_LPE_DEAD);
            }

        // join[s][r]: the forward table from s over r's representative history, read backwards (the string's order).
        // Histories that reach one reverse state match after the same camera prefixes, so any representative will do.
        out.join.assign((size_t)out.n_states * out.rev_n_states, 0u);
        out.join_any.assign(256, 0u);
        std::vector<uint32_t> history;
        for (uint32_t r = 0; r < order.size(); r++)
        {
            history.clear();
            for (uint32_t k = r; k != 0; k = parent[k]) history.push_back(via[k]);   // last event first
            for (uint32_t s = 0; s < out.n_states; s++)
            {
                uint32_t f = s;
                for (size_t k = 0; k < history.size() && f != MCRT_LPE_DEAD; k++) f = out.next[(size_t)f * n_symbols + history[k]];
                const uint32_t m = f == MCRT_LPE_DEAD ? 0u : out.accept[f];
                out.join[(size_t)s * out.rev_n_states + r] = m;
                if (m) out.join_any[s] = 1u;
            }
        }
        return std::string();
    }

    // lpeCompile without its exception guard
    static int compile(const char* const* exprs, uint32_t n, uint32_t n_groups, LpeTable& out, std::string& error)
    {
        out = LpeTable();
        if (n == 0 || !exprs) { error = "no expressions"; return MCRT_ERR_INVALID; }
        if (n > MCRT_LPE_MAX_EXPRESSIONS)
        {
            error = std::to_string(n) + " expressions, at most " + std::to_string(MCRT_LPE_MAX_EXPRESSIONS) + " (one accept bit each)";
            return MCRT_ERR_INVALID;
        }
        // parse every expression
        std::vector<Node> nodes;
        std::vector<int> roots(n);
        for (uint32_t i = 0; i < n; i++)
        {
            if (!exprs[i]) { error = "expression " + std::to_string(i) + " is null"; return MCRT_ERR_INVALID; }
            try
            {
                Parser ps(exprs[i], nodes);
                roots[i] = ps.parse();
            }
            catch (const ParseError& e)
            {
                error = "expression " + std::to_string(i) + " " + quoted(exprs[i]) + ": " + e.what + " at offset " + std::to_string(e.offset);
                return MCRT_ERR_INVALID;
            }
        }
        // number the labels: symbol MCRT_LPE_SYM_LABEL0 + k is group labels[k]
        std::vector<uint32_t> labels;
        for (const Node& nd : nodes)
            for (uint32_t g : nd.atoms.labels)
            {
                if (g >= n_groups)
                {
                    error = "label '" + std::to_string(g) + "' names no light group: " +
                            (n_groups ? "the group table has " + std::to_string(n_groups) + " groups" : std::string("there is no group table"));
                    return MCRT_ERR_INVALID;
                }
                labels.push_back(g);
            }
        std::sort(labels.begin(), labels.end());
        labels.erase(std::unique(labels.begin(), labels.end()), labels.end());
        if (labels.size() > MCRT_LPE_MAX_LABELS)
        {
            error = std::to_string(labels.size()) + " distinct labels, at most " + std::to_string(MCRT_LPE_MAX_LABELS);
            return MCRT_ERR_INVALID;
        }
        const uint32_t n_symbols = MCRT_LPE_SYM_LABEL0 + (uint32_t)labels.size();

        Nfa nfa;
        nfa.leaf_sets.resize(nodes.size());
        for (size_t id = 0; id < nodes.size(); id++)
        {
            const Node& nd = nodes[id];
            if (nd.kind != Node::SET) continue;
            SymSet s;
            for (uint32_t b = 0; b < 5; b++) if (nd.atoms.mask & (1u << b)) s.set(MCRT_LPE_SYM_RD + b);
            if (nd.atoms.mask & Atoms::B) s.set(MCRT_LPE_SYM_B);
            if (nd.atoms.mask & Atoms::C) s.set(SYM_C);
            if (nd.atoms.mask & Atoms::L) for (uint32_t k = MCRT_LPE_SYM_L; k < n_symbols; k++) s.set(k);
            for (uint32_t g : nd.atoms.labels)
                s.set(MCRT_LPE_SYM_LABEL0 + (uint32_t)(std::lower_bound(labels.begin(), labels.end(), g) - labels.begin()));
            if (nd.negated)
            {
                SymSet all;
                for (uint32_t k = 0; k < n_symbols; k++) all.set(k);
                all.set(SYM_C);
                s = all & ~s;
            }
            nfa.leaf_sets[id] = s;
        }
        int start;
        std::vector<std::pair<int, int>> ends(n);   // each expression's own start and accepting NFA state
        try
        {
            start = nfa.state();
            for (uint32_t i = 0; i < n; i++)
            {
                const std::pair<int, int> f = nfa.build(nodes, roots[i]);
                ends[i] = f;
                nfa.eps[start].push_back(f.first);
                nfa.accept[f.second] |= 1u << i;
            }
        }
        catch (const std::length_error&)
        {
            error = "the expressions' automaton exceeds " + std::to_string(MAX_NFA_STATES) + " states";
            return MCRT_ERR_UNSUPPORTED;
        }

        // subset construction over the device symbols and C (column n_symbols of dfa_next)
        const uint32_t cols = n_symbols + 1;
        std::map<std::vector<int>, uint32_t> index;
        std::vector<std::vector<int>> sets;
        std::vector<uint32_t> dfa_next, dfa_accept;
        std::vector<uint8_t> mark(nfa.eps.size(), 0);
        uint64_t steps = 0;
        auto intern = [&](std::vector<int>& set) -> uint32_t
        {
            nfa.close(set, mark);
            steps += set.size();
            auto it = index.find(set);
            if (it != index.end()) return it->second;
            const uint32_t id = (uint32_t)sets.size();
            uint32_t acc = 0;
            for (int q : set) acc |= nfa.accept[q];
            index.emplace(set, id);
            sets.push_back(set);
            dfa_accept.push_back(acc);
            dfa_next.resize(dfa_next.size() + cols, 0);
            return id;
        };
        {
            std::vector<int> s0(1, start);
            intern(s0);
        }
        for (uint32_t d = 0; d < sets.size(); d++)
        {
            if (sets.size() > MAX_DFA_STATES)
            {
                error = "the expressions need more than " + std::to_string(MAX_DFA_STATES) + " automaton states";
                return MCRT_ERR_UNSUPPORTED;
            }
            for (uint32_t col = 0; col < cols; col++)
            {
                steps += sets[d].size();
                if (steps > MAX_SUBSET_WORK)
                {
                    error = "the expressions' automaton is too large to build (more than " + std::to_string(MAX_SUBSET_WORK) +
                            " subset-construction steps)";
                    return MCRT_ERR_UNSUPPORTED;
                }
                const uint32_t sym = col < n_symbols ? col : SYM_C;
                std::vector<int> moved;
                for (int q : sets[d])
                    if (nfa.out[q] >= 0 && nfa.on[q].test(sym)) moved.push_back(nfa.out[q]);
                std::sort(moved.begin(), moved.end());
                moved.erase(std::unique(moved.begin(), moved.end()), moved.end());
                const uint32_t t = intern(moved);
                dfa_next[(size_t)d * cols + col] = t;
            }
        }

        // live: accepting, or an accepting state is reachable through device symbols (C never comes after the start)
        const uint32_t nd = (uint32_t)sets.size();
        std::vector<std::vector<uint32_t>> pred(nd);
        for (uint32_t d = 0; d < nd; d++)
            for (uint32_t col = 0; col < n_symbols; col++) pred[dfa_next[(size_t)d * cols + col]].push_back(d);
        std::vector<uint8_t> live(nd, 0);
        std::vector<uint32_t> work;
        for (uint32_t d = 0; d < nd; d++) if (dfa_accept[d]) { live[d] = 1; work.push_back(d); }
        while (!work.empty())
        {
            const uint32_t d = work.back();
            work.pop_back();
            for (uint32_t p : pred[d]) if (!live[p]) { live[p] = 1; work.push_back(p); }
        }

        // Moore's partition refinement of the live states: states with equal accept masks whose transitions lead to
        // equal classes merge (the dead states form no class). The union of many expressions that count events
        // ("C.{4}L", "C.{3,}[LB]") needs it to stay within 8 bits of state.
        std::vector<uint32_t> cls(nd, UINT32_MAX);
        size_t n_cls = 0;
        {
            std::map<uint32_t, uint32_t> by_mask;
            for (uint32_t d = 0; d < nd; d++)
                if (live[d]) cls[d] = by_mask.emplace(dfa_accept[d], (uint32_t)by_mask.size()).first->second;
            n_cls = by_mask.size();
            std::vector<uint32_t> sig(n_symbols + 1);
            for (;;)
            {
                std::map<std::vector<uint32_t>, uint32_t> by_sig;
                std::vector<uint32_t> refined(nd, UINT32_MAX);
                for (uint32_t d = 0; d < nd; d++)
                {
                    if (!live[d]) continue;
                    sig[0] = cls[d];
                    for (uint32_t col = 0; col < n_symbols; col++) sig[col + 1] = cls[dfa_next[(size_t)d * cols + col]];
                    refined[d] = by_sig.emplace(sig, (uint32_t)by_sig.size()).first->second;
                }
                const bool stable = by_sig.size() == n_cls;
                cls.swap(refined);
                n_cls = by_sig.size();
                if (stable) break;
            }
        }

        // breadth-first numbering of the classes from the state after C; order holds one DFA state of each
        const uint32_t after_c = dfa_next[n_symbols];   // row 0 (the start), column C
        std::vector<uint32_t> number(n_cls, MCRT_LPE_DEAD), order;
        if (live[after_c]) { number[cls[after_c]] = 0; order.push_back(after_c); }
        for (size_t k = 0; k < order.size(); k++)
            for (uint32_t col = 0; col < n_symbols; col++)
            {
                const uint32_t t = dfa_next[(size_t)order[k] * cols + col];
                if (!live[t] || number[cls[t]] != MCRT_LPE_DEAD) continue;
                if (order.size() >= MCRT_LPE_MAX_STATES)
                {
                    error = "the expressions need more than " + std::to_string(MCRT_LPE_MAX_STATES) +
                            " live automaton states (the path state keeps 8 bits)";
                    return MCRT_ERR_UNSUPPORTED;
                }
                number[cls[t]] = (uint32_t)order.size();
                order.push_back(t);
            }

        // nothing can match at all: one state whose every event leads to DEAD, so state 0 still exists
        out.n_states = order.empty() ? 1u : (uint32_t)order.size();
        out.n_symbols = n_symbols;
        out.next.assign((size_t)out.n_states * n_symbols, (uint8_t)MCRT_LPE_DEAD);
        out.accept.assign(256, 0u);
        for (uint32_t k = 0; k < order.size(); k++)
        {
            out.accept[k] = dfa_accept[order[k]];
            for (uint32_t col = 0; col < n_symbols; col++)
            {
                const uint32_t t = dfa_next[(size_t)order[k] * cols + col];
                out.next[(size_t)k * n_symbols + col] = (uint8_t)(live[t] ? number[cls[t]] : MCRT_LPE_DEAD);
            }
        }
        out.labels = labels;
        out.photon_error = compileReverse(nfa, ends, n_symbols, out);
        if (!out.photon_error.empty())
        {
            out.rev_n_states = 0; out.rev_start = MCRT_LPE_DEAD;
            out.rev_next.clear(); out.join.clear(); out.join_any.clear();
        }
        return MCRT_OK;
    }

    int lpeCompile(const char* const* exprs, uint32_t n, uint32_t n_groups, LpeTable& out, std::string& error)
    {
        // nothing thrown may cross the C ABI: an allocation failure is a refusal like any other limit
        try
        {
            return compile(exprs, n, n_groups, out, error);
        }
        catch (const std::exception& e)
        {
            out = LpeTable();
            error = std::string("the expressions could not be compiled: ") + e.what();
            return MCRT_ERR_UNSUPPORTED;
        }
    }
}
