//! gpu.zig -- Zig binding of libphantgpu.so (include/phant_gpu.h) for phant.
//!
//! NOT COMPILED IN THIS REPOSITORY'S CI: the build image has no Zig toolchain.  It follows the patterns phant
//! already uses for evmone (`@cImport` + `callconv(.C)`, src/blockchain/vm.zig:1-3) and is kept in step with
//! host/phant_host.hpp, which binds the same symbols and is compiled and run by tests/test_gpu_host_cpp.py.
//! Drop it at src/gpu/gpu.zig and add the build.zig lines of INTEGRATION.md section 1.
const std = @import("std");
const c = @cImport({
    @cInclude("phant_gpu.h");
});
const types = @import("../types/types.zig");
const mpt = @import("../mpt/mpt.zig");
const Allocator = std.mem.Allocator;
const Hash32 = types.Hash32;

pub const Error = error{ GpuBackend, GpuUnavailable, OutOfMemory };

pub const ProofStatus = enum(u8) { reject = 0, present = 1, absent = 2 };

pub const Gpu = struct {
    ctx: *c.phant_gpu_ctx,

    /// One context per worker thread (contexts are not re-entrant; src/main.zig:143-149 runs handlers on httpz workers).
    pub fn init(device: i32) Error!Gpu {
        if (c.phant_gpu_abi_version() != c.PHANT_GPU_ABI_VERSION) return error.GpuUnavailable;
        var cfg = std.mem.zeroes(c.phant_gpu_config);
        cfg.device = device;
        var ctx: ?*c.phant_gpu_ctx = null;
        if (c.phant_gpu_create(&ctx, &cfg) != 0) return error.GpuUnavailable; // no CUDA device: the caller keeps its CPU path
        return .{ .ctx = ctx.? };
    }

    pub fn deinit(self: *Gpu) void {
        c.phant_gpu_destroy(self.ctx);
    }

    /// hasher.keccak256 (src/crypto/hasher.zig:4-8) for many inputs: message i = msgs[off[i]..off[i+1]).
    pub fn keccak256Batch(self: *Gpu, msgs: []const u8, off: []const u64, out: []Hash32) Error!void {
        std.debug.assert(off.len == out.len + 1);
        if (c.phant_gpu_keccak256_batch(self.ctx, msgs.ptr, off.ptr, out.len, @ptrCast(out.ptr)) != 0) return error.GpuBackend;
    }

    /// == mpt.mptize (src/mpt/mpt.zig:38-45).  `list` sorted by key, as the reference asserts.
    pub fn mptize(self: *Gpu, arena: Allocator, list: []const mpt.KeyVal) Error!Hash32 {
        var keys = std.ArrayList(u8).init(arena);
        var vals = std.ArrayList(u8).init(arena);
        var key_off = try arena.alloc(u32, list.len + 1);
        var val_off = try arena.alloc(u64, list.len + 1);
        key_off[0] = 0;
        val_off[0] = 0;
        for (list, 0..) |kv, i| {
            var j: usize = 0;
            while (j + 1 < kv.nibbles.len) : (j += 2) try keys.append((kv.nibbles[j] << 4) | kv.nibbles[j + 1]); // KeyVal.init always makes nibble pairs
            try vals.appendSlice(kv.value);
            key_off[i + 1] = @intCast(keys.items.len);
            val_off[i + 1] = vals.items.len;
        }
        var root: Hash32 = undefined;
        if (c.phant_gpu_mpt_root(self.ctx, keys.items.ptr, key_off.ptr, vals.items.ptr, val_off.ptr, list.len, &root) != 0) return error.GpuBackend;
        return root;
    }

    /// The body of the missing StateDB.root() (hook: src/blockchain/blockchain.zig:83-85).
    pub fn stateRoot(self: *Gpu, accounts: *const c.phant_gpu_accounts) Error!Hash32 {
        var root: Hash32 = undefined;
        if (c.phant_gpu_state_root(self.ctx, accounts, &root) != 0) return error.GpuBackend;
        return root;
    }

    /// StateDB.root() sharded over GPUs: hashes of the 16 subtrees under the account trie's root branch for the accounts
    /// handed in (those whose keccak(addr) top nibble this rank owns) and the mask of populated slots.
    pub fn stateSubtreeRoots(self: *Gpu, accounts: *const c.phant_gpu_accounts, out_roots: *[16 * 32]u8) Error!u32 {
        var mask: u32 = 0;
        if (c.phant_gpu_state_subtree_roots(self.ctx, accounts, out_roots, &mask) != 0) return error.GpuBackend;
        return mask;
    }

    /// The body of the TODO at src/engine_api/execution_payload.zig:177-178.  Accept / reject is data.
    pub fn verifyProofs(self: *Gpu, batch: *const c.phant_gpu_proof_batch, accept_bitmap: []u64, status: ?[]u8) Error!void {
        std.debug.assert(accept_bitmap.len * 64 >= batch.n_proofs);
        const st: ?[*]u8 = if (status) |s| s.ptr else null;
        if (c.phant_gpu_verify_proofs(self.ctx, batch, accept_bitmap.ptr, st, null, null) != 0) return error.GpuBackend;
    }

    /// The same check for a witness that is an unordered SET of trie nodes (status 3 = a node on the key's path is missing).
    pub fn verifyWitness(self: *Gpu, witness: *const c.phant_gpu_witness, accept_bitmap: []u64, status: ?[]u8) Error!void {
        std.debug.assert(accept_bitmap.len * 64 >= witness.n_keys);
        const st: ?[*]u8 = if (status) |s| s.ptr else null;
        if (c.phant_gpu_verify_witness(self.ctx, witness, accept_bitmap.ptr, st, null, null) != 0) return error.GpuBackend;
    }

    /// Pre-state reads: what the witness's node set proves about the accounts and slots a block touches, decoded (nonce,
    /// balance, storage root, code index, slot values), with every slot walked from its account's proven storage root on the
    /// device.  The first call of the stateless handler (StatelessPayloadStatusV1, execution_payload.zig:20-25, TODO at
    /// :177-178): the values fill the StateDB the block executes against (src/state/types.zig:13-33).
    pub fn readState(self: *Gpu, reads: *const c.phant_gpu_state_reads, values: *c.phant_gpu_state_values) Error!void {
        if (c.phant_gpu_read_state(self.ctx, reads, values) != 0) return error.GpuBackend;
    }

    /// State transition roots: each block's post-state root from the witness's node set, its parent root and the diff execution
    /// wrote (StatelessPayloadStatusV1.state_root, execution_payload.zig:20-25; the check at blockchain.zig:83-85).  status[b] =
    /// 1 root computed, 0 a node breaks the rules, 3 the witness lacks a node; roots are zero unless the status is 1.
    pub fn transitionRoots(self: *Gpu, t: *const c.phant_gpu_transition, diff: *const c.phant_gpu_state_diff, post_roots: []Hash32, status: []u8) Error!void {
        std.debug.assert(post_roots.len == t.n_blocks and status.len == t.n_blocks);
        if (c.phant_gpu_transition_roots(self.ctx, t, diff, @ptrCast(post_roots.ptr), status.ptr, null) != 0) return error.GpuBackend;
    }

    /// Many tries in one forest build: the transaction / receipt / withdrawal tries of a block or of a range of blocks
    /// (src/blockchain/blockchain.zig:200-203).  Trie t = items [seg_off[t], seg_off[t+1]) of the CSR arrays.
    pub fn mptRoots(self: *Gpu, keys: []const u8, key_off: []const u32, vals: []const u8, val_off: []const u64, seg_off: []const u32, out_roots: []Hash32) Error!void {
        std.debug.assert(seg_off.len == out_roots.len + 1);
        if (c.phant_gpu_mpt_roots(self.ctx, keys.ptr, key_off.ptr, vals.ptr, val_off.ptr, seg_off.ptr, out_roots.len, @ptrCast(out_roots.ptr)) != 0)
            return error.GpuBackend;
    }

    /// The tail of TxSigner.get_sender (src/signer/signer.zig:78-79) for a whole block: sigs65[i] = r || s || recid over
    /// hashes[i]; ok[i] == 0 where erecover would have failed.
    pub fn recoverSenders(self: *Gpu, hashes: []const Hash32, sigs65: []const [65]u8, addresses: [][20]u8, ok: []u8) Error!void {
        std.debug.assert(hashes.len == sigs65.len and hashes.len == addresses.len and hashes.len == ok.len);
        if (c.phant_gpu_ecrecover_batch(self.ctx, @ptrCast(hashes.ptr), @ptrCast(sigs65.ptr), hashes.len, null, @ptrCast(addresses.ptr), ok.ptr) != 0)
            return error.GpuBackend;
    }

    // ---- multi-GPU: one Gpu (context) per device, one worker thread each (src/main.zig:143-149) ----

    /// One process driving several devices: rank i = gpus[i].  NCCL is loaded inside libphantgpu.so.
    pub fn commInitLocal(gpus: []Gpu, arena: Allocator) Error!void {
        const ctxs = try arena.alloc(?*c.phant_gpu_ctx, gpus.len);
        for (gpus, 0..) |g, i| ctxs[i] = g.ctx;
        if (c.phant_gpu_comm_init_local(@ptrCast(ctxs.ptr), @intCast(gpus.len)) != 0) return error.GpuBackend;
    }

    /// One process per device: rank 0 creates the id (phant_gpu_comm_get_unique_id) and hands it to the others.
    pub fn commInit(self: *Gpu, id: *const [c.PHANT_GPU_COMM_ID_BYTES]u8, rank: i32, world: i32) Error!void {
        if (c.phant_gpu_comm_init(self.ctx, id, rank, world) != 0) return error.GpuBackend;
    }

    /// Optional, collective: map every rank's bitmap region into every other rank (NVLink); equal-shard device-pointer calls of
    /// verifyProofsSharded then gather inside the walk kernel.  error.GpuBackend = not possible here, NCCL stays in use.
    pub fn commEnablePeer(self: *Gpu, max_proofs: u64) Error!void {
        if (c.phant_gpu_comm_enable_peer(self.ctx, max_proofs) != 0) return error.GpuBackend;
    }

    /// verifyProofs for this rank's shard of a batch of n_global proofs (phant_gpu_shard_range); on return global_bitmap
    /// (phant_gpu_sharded_bitmap_words(n_global, world) words) holds every rank's accept bits.
    pub fn verifyProofsSharded(self: *Gpu, local: *const c.phant_gpu_proof_batch, n_global: u64, global_bitmap: []u64, status: ?[]u8) Error!void {
        const st: ?[*]u8 = if (status) |s| s.ptr else null;
        if (c.phant_gpu_verify_proofs_sharded(self.ctx, local, n_global, global_bitmap.ptr, st, null, null) != 0) return error.GpuBackend;
    }

    /// StateDB.root() across GPUs: `mine` = the accounts whose keccak(address) top nibble this rank owns
    /// (phant_gpu_nibble_owner); every rank gets the same root.
    pub fn stateRootSharded(self: *Gpu, mine: *const c.phant_gpu_accounts) Error!Hash32 {
        var root: Hash32 = undefined;
        if (c.phant_gpu_state_root_sharded(self.ctx, mine, &root) != 0) return error.GpuBackend;
        return root;
    }

    // ---- resident state trie: StateDB.root() after a block costs the dirty accounts, not a rebuild ----

    pub const ResidentTrie = struct {
        t: *c.phant_gpu_trie,

        /// kind 1: sparse secure trie, initially empty; feed it the genesis / snapshot accounts with one `apply`.
        pub fn open(gpu: *Gpu) Error!ResidentTrie {
            var desc = std.mem.zeroes(c.phant_gpu_trie_desc);
            desc.kind = 1;
            var t: ?*c.phant_gpu_trie = null;
            if (c.phant_gpu_trie_open(gpu.ctx, &desc, &t) != 0) return error.GpuBackend;
            return .{ .t = t.? };
        }
        /// upsert (keccak(address) -> rlp(account)); an empty value deletes the account.  Returns the new state root.
        pub fn apply(self: *ResidentTrie, keys32: []const u8, vals: []const u8, val_off: []const u32) Error!Hash32 {
            var root: Hash32 = undefined;
            if (c.phant_gpu_trie_update(self.t, keys32.ptr, vals.ptr, val_off.ptr, val_off.len - 1, &root) != 0) return error.GpuBackend;
            return root;
        }
        pub fn close(self: *ResidentTrie) void {
            c.phant_gpu_trie_close(self.t);
        }
    };

    /// The account trie AND every storage trie resident (DESIGN.md §4.3c): load the snapshot with one `apply`, then per block
    /// pass the journal's touched accounts and dirty slots (hashed keys); no storage root is computed on the host.
    pub const ResidentState = struct {
        s: *c.phant_gpu_resident_state,

        pub fn open(gpu: *Gpu) Error!ResidentState {
            var s: ?*c.phant_gpu_resident_state = null;
            if (c.phant_gpu_resident_state_open(gpu.ctx, &s) != 0) return error.GpuBackend;
            return .{ .s = s.? };
        }
        /// storage_roots32: null, or 32 bytes per listed account (zero for deleted ones).  Returns the new state root.
        pub fn apply(self: *ResidentState, diff: *const c.phant_gpu_state_diff, storage_roots32: ?[]u8) Error!Hash32 {
            var root: Hash32 = undefined;
            const sr: [*c]u8 = if (storage_roots32) |b| b.ptr else null;
            if (c.phant_gpu_resident_state_apply(self.s, diff, &root, sr) != 0) return error.GpuBackend;
            return root;
        }
        pub fn root(self: *ResidentState) Error!Hash32 {
            var r: Hash32 = undefined;
            if (c.phant_gpu_resident_state_root(self.s, &r) != 0) return error.GpuBackend;
            return r;
        }
        /// Keep what undoes each of the last `depth` applies on the device (0: none, the default; at most 1024).
        pub fn setJournal(self: *ResidentState, depth: u32) Error!void {
            if (c.phant_gpu_resident_state_set_journal(self.s, depth) != 0) return error.GpuBackend;
        }
        /// Undo the last n applies, newest first (a block whose root did not match its header, or the blocks a reorg
        /// leaves).  Returns the root before the oldest of them.
        pub fn revert(self: *ResidentState, n: u32) Error!Hash32 {
            var r: Hash32 = undefined;
            if (c.phant_gpu_resident_state_revert(self.s, n, &r) != 0) return error.GpuBackend;
            return r;
        }
        /// The execution witness of `diff` from the state as it is now (the state is not changed): the pre-state trie nodes
        /// the block reads or changes, each once, ordered by digest, as one arena and n + 1 offsets in `arena`.
        pub fn witness(self: *ResidentState, arena: Allocator, diff: *const c.phant_gpu_state_diff) Error!struct { nodes: []u8, node_off: []u64 } {
            var size: c.phant_gpu_witness_size = undefined;
            if (c.phant_gpu_resident_state_witness(self.s, diff, &size) != 0) return error.GpuBackend;
            const nodes = arena.alloc(u8, @intCast(size.nodes_bytes + 1)) catch return error.OutOfMemory;
            const off = arena.alloc(u64, @intCast(size.n_nodes + 1)) catch return error.OutOfMemory;
            if (c.phant_gpu_resident_state_witness_copy(self.s, nodes.ptr, off.ptr) != 0) return error.GpuBackend;
            return .{ .nodes = nodes[0..@intCast(size.nodes_bytes)], .node_off = off };
        }
        pub fn close(self: *ResidentState) void {
            c.phant_gpu_resident_state_close(self.s);
        }
    };

    /// Receipt.calculateLogsBloom (src/types/receipt.zig:37-48) for all receipts of a block.
    pub fn logsBlooms(self: *Gpu, items: []const u8, item_off: []const u64, bloom_of_item: []const u32, blooms: []types.LogsBloom) Error!void {
        if (c.phant_gpu_logs_bloom(self.ctx, items.ptr, item_off.ptr, bloom_of_item.ptr, bloom_of_item.len, blooms.len, @ptrCast(blooms.ptr)) != 0)
            return error.GpuBackend;
    }
};

/// Flatten phant's StateDB (src/state/statedb.zig:16-30) into the SoA the library takes and return the state root.
pub fn stateDbRoot(gpu: *Gpu, arena: Allocator, statedb: anytype) Error!Hash32 {
    var addr = std.ArrayList(u8).init(arena);
    var nonce = std.ArrayList(u64).init(arena);
    var balance = std.ArrayList(u8).init(arena);
    var code = std.ArrayList(u8).init(arena);
    var code_off = std.ArrayList(u64).init(arena);
    var slot_keys = std.ArrayList(u8).init(arena);
    var slot_vals = std.ArrayList(u8).init(arena);
    var slot_off = std.ArrayList(u64).init(arena);
    try code_off.append(0);
    try slot_off.append(0);
    var it = statedb.db.iterator();
    while (it.next()) |entry| {
        try addr.appendSlice(&entry.key_ptr.*);
        try nonce.append(entry.value_ptr.nonce);
        var be: [32]u8 = undefined;
        std.mem.writeInt(u256, &be, entry.value_ptr.balance, .big);
        try balance.appendSlice(&be);
        try code.appendSlice(entry.value_ptr.code);
        try code_off.append(code.items.len);
        var sit = entry.value_ptr.storage.iterator();
        while (sit.next()) |s| {
            std.mem.writeInt(u256, &be, s.key_ptr.*, .big);
            try slot_keys.appendSlice(&be);
            try slot_vals.appendSlice(&s.value_ptr.*);
        }
        try slot_off.append(slot_keys.items.len / 32);
    }
    const table = c.phant_gpu_accounts{
        .n_accounts = nonce.items.len,
        .addr20 = addr.items.ptr,
        .nonce = nonce.items.ptr,
        .balance32 = balance.items.ptr,
        .code = code.items.ptr,
        .code_off = code_off.items.ptr,
        .slot_keys32 = slot_keys.items.ptr,
        .slot_vals32 = slot_vals.items.ptr,
        .slot_off = slot_off.items.ptr,
    };
    return gpu.stateRoot(&table);
}
