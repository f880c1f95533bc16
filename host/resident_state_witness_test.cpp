// resident_state_witness_test.cpp -- witnesses from the resident world state in C++ (phant_host.hpp:
// ResidentStateTrie::witness), checked with engine_api::transitionRoot.  Reads cases from the file named on the command line
// (written by tests/test_gpu_host_cpp_resident_state_witness.py from the fixture states), one line each:
//   case <pre state root hex> <post state root hex>
//   pre <address hex> <nonce> <balance hex, 32 bytes> <code hex or -> | pslot <address hex> <slot hex, 32 bytes> <value hex>
//   acct <address hex> <nonce> <balance hex, 32 bytes> <code hex or -> | del <address hex>
//   slot <address hex> <slot number hex, 32 bytes> <new value hex, 32 bytes>
//   end
// Per case: the pre-state is loaded and gives the pre root; the block's witness from it, with the pre root and the block's
// changes, gives the header's post root with status 1 through transitionRoot; the apply then gives the same root.  Prints
// "ALL OK".
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
    Hash32 pre_root{}, post{};
    std::map<Address, state::AccountState> pre, live;
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
    state::ResidentStateTrie st(g);
    std::map<Address, const state::AccountState*> load;
    for (const auto& [a, s] : c.pre) load[a] = &s;
    if (!load.empty() && st.apply(load) != c.pre_root) { std::cout << "case " << n << ": pre root mismatch\n"; return 1; }
    const std::vector<Bytes> nodes = st.witness(c.touched(), c.slots);
    if (st.root() != c.pre_root) { std::cout << "case " << n << ": the witness changed the state\n"; return 1; }
    if (!c.live.empty() || !c.gone.empty()) {
        const engine_api::TransitionResult r = engine_api::transitionRoot(g, c.pre_root, nodes, c.touched(), c.slots);
        if (r.status != 1 || r.root != c.post) { std::cout << "case " << n << ": status " << int(r.status) << ", root mismatch\n"; return 1; }
    }
    if (st.apply(c.touched(), c.slots) != c.post) { std::cout << "case " << n << ": apply root mismatch\n"; return 1; }
    return 0;
}

int main(int argc, char** argv)
{
    if (argc != 2) { std::cerr << "usage: resident_state_witness_test CASES\n"; return 2; }
    std::ifstream f(argv[1]);
    Gpu g(0);
    std::string line;
    Case c;
    int n = 0, bad = 0;
    while (std::getline(f, line)) {
        std::istringstream ls(line);
        std::string kind, a, b, x, y;
        ls >> kind >> a >> b >> x >> y;
        if (kind == "case") { c = Case{}; c.pre_root = fixed<32>(a); c.post = fixed<32>(b); }
        else if (kind == "pre" || kind == "acct") {
            state::AccountState s;
            s.nonce = std::stoull(b);
            s.balance = fixed<32>(x);
            if (y != "-") s.code = unhex(y);
            (kind == "pre" ? c.pre : c.live)[fixed<20>(a)] = s;
        } else if (kind == "pslot") c.pre[fixed<20>(a)].storage[fixed<32>(b)] = fixed<32>(x);
        else if (kind == "del") c.gone.insert(fixed<20>(a));
        else if (kind == "slot") c.slots[fixed<20>(a)][fixed<32>(b)] = fixed<32>(x);
        else if (kind == "end") { bad += run(g, c, n); ++n; }
    }
    if (n == 0 || bad) { std::cout << bad << " of " << n << " cases failed\n"; return 1; }
    std::cout << n << " cases\nALL OK\n";
    return 0;
}
