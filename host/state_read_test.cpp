// state_read_test.cpp -- the C++ pre-state factory (phant_host.hpp: engine_api::readPreState / stateDBFromWitness) through the
// C ABI.  Reads cases from the file named on the command line (written by tests/test_gpu_host_cpp_state_reads.py from the
// fixture states), one line each:
//   case <state root hex> <expected root of what is read hex>
//   node <hex> | code <hex> | addr <hex> | absent <hex> | slot <address hex> <slot number hex, 32 bytes>
//   end
// Per case: the StateDB built from the witness has the expected state root, absent addresses are status 2 and not in it; the
// same witness without its codes, and without one of its nodes, is refused with IncompleteWitness.  Prints "ALL OK".
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
static std::string hex(const Hash32& h)
{
    char buf[65];
    for (int i = 0; i < 32; ++i) snprintf(buf + 2 * i, 3, "%02x", h[i]);
    return std::string(buf, 64);
}

struct Case {
    Hash32 root{}, expect{};
    std::vector<Bytes> nodes, codes;
    std::vector<Address> addrs, absent;
    std::vector<engine_api::SlotRead> slots;
};

static bool refused(Gpu& g, const Case& c, const std::vector<Bytes>& nodes, const std::vector<Bytes>& codes)
{
    std::vector<Address> all = c.addrs;
    all.insert(all.end(), c.absent.begin(), c.absent.end());
    try {
        engine_api::stateDBFromWitness(g, c.root, nodes, codes, all, c.slots);
    } catch (const engine_api::IncompleteWitness&) {
        return true;
    }
    return false;
}

static int run(Gpu& g, const Case& c, int n)
{
    std::vector<Address> all = c.addrs;
    all.insert(all.end(), c.absent.begin(), c.absent.end());
    const engine_api::PreState pre = engine_api::readPreState(g, c.root, c.nodes, c.codes, all, c.slots);
    if (!pre.complete()) { std::cout << "case " << n << ": incomplete\n"; return 1; }
    for (const Address& a : c.absent)
        if (pre.account_status.at(a) != 2 || pre.statedb.db.count(a)) { std::cout << "case " << n << ": absent account\n"; return 1; }
    const state::StateDB db = engine_api::stateDBFromWitness(g, c.root, c.nodes, c.codes, all, c.slots);
    if (db.db.size() != c.addrs.size()) { std::cout << "case " << n << ": account count\n"; return 1; }
    const Hash32 r = db.root(g);
    if (r != c.expect) { std::cout << "case " << n << ": root " << hex(r) << " != " << hex(c.expect) << "\n"; return 1; }
    bool has_code = false;
    for (const auto& [a, acc] : db.db) has_code = has_code || !acc.code.empty();
    if (has_code && !refused(g, c, c.nodes, {})) { std::cout << "case " << n << ": missing code accepted\n"; return 1; }
    // drop the last node (a leaf of some proof): some read lacks a node
    std::vector<Bytes> fewer(c.nodes.begin(), c.nodes.end() - 1);
    if (!refused(g, c, fewer, c.codes)) { std::cout << "case " << n << ": missing node accepted\n"; return 1; }
    return 0;
}

int main(int argc, char** argv)
{
    if (argc != 2) { std::cerr << "usage: state_read_test CASES\n"; return 2; }
    std::ifstream f(argv[1]);
    Gpu g(0);
    std::string line;
    Case c;
    int n = 0, bad = 0;
    while (std::getline(f, line)) {
        std::istringstream ls(line);
        std::string kind, a, b;
        ls >> kind >> a >> b;
        if (kind == "case") { c = Case{}; c.root = fixed<32>(a); c.expect = fixed<32>(b); }
        else if (kind == "node") c.nodes.push_back(unhex(a));
        else if (kind == "code") c.codes.push_back(unhex(a));
        else if (kind == "addr") c.addrs.push_back(fixed<20>(a));
        else if (kind == "absent") c.absent.push_back(fixed<20>(a));
        else if (kind == "slot") c.slots.push_back({fixed<20>(a), fixed<32>(b)});
        else if (kind == "end") { bad += run(g, c, n); ++n; }
    }
    if (n == 0 || bad) { std::cout << bad << " of " << n << " cases failed\n"; return 1; }
    std::cout << n << " cases\nALL OK\n";
    return 0;
}
