// transition_test.cpp -- the C++ transition root (phant_host.hpp: engine_api::transitionRoot) through the C ABI.  Reads cases
// from the file named on the command line (written by tests/test_gpu_host_cpp_transition.py from the fixture states), one
// line each:
//   case <parent state root hex> <post state root hex>
//   node <hex> | acct <address hex> <nonce> <balance hex, 32 bytes> <code hex or -> | del <address hex>
//   slot <address hex> <slot number hex, 32 bytes> <new value hex, 32 bytes>
//   end
// Per case: the root is the header's post root with status 1; a block with one nonce changed gives another root; the
// witness without its last node (the root node of the account trie) gives status 3.  Prints "ALL OK".
#include "phant_host.hpp"

#include <cstdio>
#include <fstream>
#include <iostream>
#include <sstream>

using namespace phant;

static Bytes unhex(const std::string& s)
{
    Bytes b(s.size() / 2);
    for (size_t i = 0; i < b.size(); ++i) b[i] = (uint8_t)std::stoi(s.substr(2 * i, 2), nullptr, 16);
    return b;
}
template <size_t N> static std::array<uint8_t, N> fixed(const std::string& s)
{
    const Bytes b = unhex(s);
    if (b.size() != N) throw std::invalid_argument("bad length: " + s);
    std::array<uint8_t, N> a;
    std::copy(b.begin(), b.end(), a.begin());
    return a;
}

struct Case {
    Hash32 parent{}, post{};
    std::vector<Bytes> nodes;
    std::map<Address, state::AccountState> live;
    std::set<Address> gone;
    state::HashedDiff::SlotChanges slots;
    std::map<Address, const state::AccountState*> touched() const
    {
        std::map<Address, const state::AccountState*> t;
        for (const auto& [a, s] : live) t[a] = &s;
        for (const Address& a : gone) t[a] = nullptr;
        return t;
    }
};

static int run(Gpu& g, Case& c, int n)
{
    const engine_api::TransitionResult r = engine_api::transitionRoot(g, c.parent, c.nodes, c.touched(), c.slots);
    if (r.status != 1 || r.root != c.post) { std::cout << "case " << n << ": status " << int(r.status) << ", root mismatch\n"; return 1; }
    if (!c.live.empty()) {
        c.live.begin()->second.nonce += 1;
        const engine_api::TransitionResult t = engine_api::transitionRoot(g, c.parent, c.nodes, c.touched(), c.slots);
        c.live.begin()->second.nonce -= 1;
        if (t.status != 1 || t.root == c.post) { std::cout << "case " << n << ": a changed nonce kept the root\n"; return 1; }
    }
    if (c.nodes.size() > 1 && !(c.live.empty() && c.gone.empty())) {
        const std::vector<Bytes> fewer(c.nodes.begin(), c.nodes.end() - 1);
        const engine_api::TransitionResult m = engine_api::transitionRoot(g, c.parent, fewer, c.touched(), c.slots);
        if (m.status != 3 || m.root != Hash32{}) { std::cout << "case " << n << ": missing root node gave status " << int(m.status) << "\n"; return 1; }
    }
    return 0;
}

int main(int argc, char** argv)
{
    if (argc != 2) { std::cerr << "usage: transition_test CASES\n"; return 2; }
    std::ifstream f(argv[1]);
    Gpu g(0);
    std::string line;
    Case c;
    int n = 0, bad = 0;
    while (std::getline(f, line)) {
        std::istringstream ls(line);
        std::string kind, a, b, x, y;
        ls >> kind >> a >> b >> x >> y;
        if (kind == "case") { c = Case{}; c.parent = fixed<32>(a); c.post = fixed<32>(b); }
        else if (kind == "node") c.nodes.push_back(unhex(a));
        else if (kind == "acct") {
            state::AccountState s;
            s.nonce = std::stoull(b);
            s.balance = fixed<32>(x);
            if (y != "-") s.code = unhex(y);
            c.live[fixed<20>(a)] = s;
        } else if (kind == "del") c.gone.insert(fixed<20>(a));
        else if (kind == "slot") c.slots[fixed<20>(a)][fixed<32>(b)] = fixed<32>(x);
        else if (kind == "end") { bad += run(g, c, n); ++n; }
    }
    if (n == 0 || bad) { std::cout << bad << " of " << n << " cases failed\n"; return 1; }
    std::cout << n << " cases\nALL OK\n";
    return 0;
}
