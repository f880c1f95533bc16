// resident_state_revert_test.cpp -- undo through the C++ mirror (phant_host.hpp: ResidentStateTrie::setJournal / revert):
// blocks are applied in the incremental form and checked against StateDB::root() (a full S rebuild); a block with a wrong
// balance is reverted as a client would on a state-root mismatch, then the last blocks are reverted as in a reorg and another
// branch is applied.  Prints "ALL OK".
#include "phant_host.hpp"

#include <cstdio>
#include <iostream>
#include <random>

using namespace phant;

static int failures = 0;
static void expect(const Hash32& got, const Hash32& want, const std::string& what)
{
    if (got != want) { std::cout << "FAIL " << what << "\n"; ++failures; }
}

int main()
{
    Gpu g;
    std::mt19937_64 rng(9);
    auto word = [&]() { std::array<uint8_t, 32> w{}; for (auto& b : w) b = (uint8_t)rng(); return w; };
    auto addr = [&]() { Address a; for (auto& b : a) b = (uint8_t)rng(); return a; };
    state::StateDB db;
    std::vector<Address> addrs;
    for (int i = 0; i < 200; ++i) {
        const Address a = addr();
        addrs.push_back(a);
        auto& acc = db.db[a];
        acc.nonce = i;
        acc.balance[31] = (uint8_t)i;
        for (int s = 0; s < i % 25; ++s) acc.storage[word()] = word();
    }
    state::ResidentStateTrie rt(g);
    rt.setJournal(8);
    std::map<Address, const state::AccountState*> all;
    for (const auto& [a, acc] : db.db) all[a] = &acc;
    expect(rt.apply(all), db.root(g), "load");

    // one block: slot writes and deletes, a balance change, a destroyed account, a created one; `db` is changed in place
    auto run_block = [&](int blk) {
        std::map<Address, const state::AccountState*> touched;
        state::ResidentStateTrie::SlotChanges changed;
        auto write = [&](const Address& a, const std::array<uint8_t, 32>& k, const std::array<uint8_t, 32>& v) {
            auto& acc = db.db[a];
            if (v == std::array<uint8_t, 32>{}) acc.storage.erase(k); else acc.storage[k] = v;
            changed[a][k] = v;
        };
        for (int s = 0; s < 300; ++s) write(addrs[1], word(), word());
        for (int i = 10; i < 30; ++i) {
            auto& acc = db.db[addrs[i]];
            if (acc.storage.empty()) continue;
            const auto k = acc.storage.begin()->first; // a copy: a delete erases the map node the key lives in
            write(addrs[i], k, (i + blk) % 2 ? word() : std::array<uint8_t, 32>{});
        }
        for (const auto& [a, s] : changed) touched[a] = &db.db[a];
        db.db[addrs[40 + blk]].balance[0] ^= 1;
        touched[addrs[40 + blk]] = &db.db[addrs[40 + blk]];
        const Address gone = addrs[100 + blk];
        if (db.db.count(gone)) { db.db.erase(gone); touched[gone] = nullptr; }
        const Address fresh = addr();
        db.db[fresh].nonce = 1;
        write(fresh, word(), word());
        touched[fresh] = &db.db[fresh];
        return rt.apply(touched, changed);
    };

    std::vector<state::StateDB> states{db};
    std::vector<Hash32> roots{db.root(g)};
    for (int blk = 0; blk < 5; ++blk) {
        const Hash32 got = run_block(blk); // before db.root(): the block changes `db`
        expect(got, db.root(g), "block " + std::to_string(blk));
        // the next block arrives with a wrong balance for one account: its root does not match, so it is reverted
        state::AccountState wrong = db.db[addrs[70]];
        wrong.balance[5] ^= 0x10;
        const Hash32 bad = rt.apply({{addrs[70], &wrong}});
        if (bad == db.root(g)) { std::cout << "FAIL tampered block " << blk << " has the true root\n"; ++failures; }
        expect(rt.revert(1), db.root(g), "revert of the invalid block " + std::to_string(blk));
        states.push_back(db);
        roots.push_back(db.root(g));
    }
    expect(rt.root(), roots.back(), "root() after the reverts");

    // a reorg of depth 3: back to the state after block 1, then another branch of three blocks
    expect(rt.revert(3), roots[2], "revert(3)");
    db = states[2];
    for (int blk = 10; blk < 13; ++blk) {
        const Hash32 got = run_block(blk);
        expect(got, db.root(g), "branch block " + std::to_string(blk));
    }
    expect(rt.root(), db.root(g), "root()");
    if (failures) return 1;
    std::cout << "ALL OK\n";
    return 0;
}
