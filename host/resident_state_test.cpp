// resident_state_test.cpp -- StateDB.root() block after block through the C++ mirror (phant_host.hpp: ResidentStateTrie) with
// only the changed slots sent (the incremental apply), checked against StateDB::root() (a full S rebuild) after every block.
// Blocks write and delete slots, grow one account past 256 and 4,096 slots (its storage depth changes), create, destroy and
// re-create accounts.  Prints "ALL OK".
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
    std::mt19937_64 rng(7);
    auto word = [&]() { std::array<uint8_t, 32> w{}; for (auto& b : w) b = (uint8_t)rng(); return w; };
    auto addr = [&]() { Address a; for (auto& b : a) b = (uint8_t)rng(); return a; };
    state::StateDB db;
    std::vector<Address> addrs;
    for (int i = 0; i < 300; ++i) {
        const Address a = addr();
        addrs.push_back(a);
        auto& acc = db.db[a];
        acc.nonce = i;
        acc.balance[31] = (uint8_t)i;
        if (i % 3 == 0) acc.code = {0x60, (uint8_t)i, 0x00};
        for (int s = 0; s < i % 20; ++s) acc.storage[word()] = word();
    }
    state::ResidentStateTrie rt(g);
    std::map<Address, const state::AccountState*> all;
    for (const auto& [a, acc] : db.db) all[a] = &acc;
    expect(rt.apply(all), db.root(g), "load");
    const Address grower = addrs[1];
    for (int blk = 0; blk < 6; ++blk) {
        std::map<Address, const state::AccountState*> touched;
        state::ResidentStateTrie::SlotChanges changed;
        auto write = [&](const Address& a, const std::array<uint8_t, 32>& k, const std::array<uint8_t, 32>& v) {
            auto& acc = db.db[a];
            if (v == std::array<uint8_t, 32>{}) acc.storage.erase(k); else acc.storage[k] = v;
            changed[a][k] = v;
        };
        // the growing account: 300 more slots per block (L 0 -> 1), then 4,000 in block 3 (L 2)
        for (int s = 0; s < (blk == 3 ? 4000 : 300); ++s) write(grower, word(), word());
        // updates and deletes of existing slots, a zero written to an absent slot
        for (int i = 10; i < 40; ++i) {
            auto& acc = db.db[addrs[i]];
            if (acc.storage.empty()) continue;
            const auto k = acc.storage.begin()->first;
            write(addrs[i], k, (i + blk) % 2 ? word() : std::array<uint8_t, 32>{});
        }
        write(addrs[50], word(), std::array<uint8_t, 32>{});
        for (const auto& [a, s] : changed) touched[a] = &db.db[a];
        // field changes without slot changes
        db.db[addrs[60 + blk]].balance[0] ^= 1;
        touched[addrs[60 + blk]] = &db.db[addrs[60 + blk]];
        // a destroyed account, a created one, and (block 4) one destroyed and re-created: old slots gone, new ones written
        const Address gone = addrs[100 + blk];
        db.db.erase(gone);
        touched[gone] = nullptr;
        const Address fresh = addr();
        db.db[fresh].nonce = 1;
        for (int s = 0; s < 5; ++s) write(fresh, word(), word());
        touched[fresh] = &db.db[fresh];
        expect(rt.apply(touched, changed), db.root(g), "block " + std::to_string(blk));
        if (blk == 4) {
            const Address again = addrs[200];
            db.db[again] = state::AccountState{};
            db.db[again].nonce = 3;
            std::map<Address, const state::AccountState*> t2{{again, &db.db[again]}};
            state::ResidentStateTrie::SlotChanges c2;
            const auto k = word(), v = word();
            db.db[again].storage[k] = v;
            expect(rt.apply(t2), db.root(g), "re-created (whole storage form)");
            c2[again][k] = std::array<uint8_t, 32>{};
            db.db[again].storage.erase(k);
            expect(rt.apply(t2, c2), db.root(g), "re-created, slot deleted");
            // destroyed and created again in one block, in the incremental form: old slots dropped, one new slot written
            const Address phoenix = addrs[201];
            db.db[phoenix] = state::AccountState{};
            db.db[phoenix].balance[31] = 9;
            const auto k3 = word(), v3 = word();
            db.db[phoenix].storage[k3] = v3;
            state::ResidentStateTrie::SlotChanges c3;
            c3[phoenix][k3] = v3;
            expect(rt.apply({{phoenix, &db.db[phoenix]}}, c3, {phoenix}), db.root(g), "re-created, incremental form");
        }
    }
    expect(rt.root(), db.root(g), "root()");
    if (failures) return 1;
    std::cout << "ALL OK\n";
    return 0;
}
