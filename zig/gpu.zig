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

    /// Range proofs (snap GetAccountRange / GetStorageRanges): each range's entries against its root, with the boundary
    /// proofs of its origin and last key in one node set, many ranges per call.  status[r] = 1 the entries are exactly the
    /// trie's contents in [origin, last] (with PHANT_GPU_RANGE_WHOLE: the whole trie), 0 they are not, 3 a node is missing;
    /// more[r] = 1 when an accepted range's trie holds a key after its last entry (null: status only).
    pub fn verifyRanges(self: *Gpu, in: *const c.phant_gpu_range_proofs, status: []u8, more: ?[]u8) Error!void {
        std.debug.assert(status.len == in.n_ranges and (more == null or more.?.len == in.n_ranges));
        const more_ptr: ?[*]u8 = if (more) |m| m.ptr else null;
        if (c.phant_gpu_verify_ranges(self.ctx, in, status.ptr, more_ptr) != 0) return error.GpuBackend;
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
        /// Account and storage proofs (eth_getProof) under the state as it is now (the state is not changed): proof p < n
        /// is account p, proof n + j slot j; chain p is node_index[proof_first[p] .. proof_first[p+1]) into the node set,
        /// root first.  Every array is allocated in `arena`.  Not compiled: the build has no Zig toolchain.
        pub fn prove(self: *ResidentState, arena: Allocator, req: *const c.phant_gpu_proof_request) Error!struct {
            nodes: []u8,
            node_off: []u64,
            node_index: []u64,
            proof_first: []u64,
            roots32: []u8,
            status: []u8,
            nonce: []u64,
            balance32: []u8,
            storage_root32: []u8,
            code_hash32: []u8,
            slot_vals32: []u8,
        } {
            var size: c.phant_gpu_proof_size = undefined;
            if (c.phant_gpu_resident_state_prove(self.s, req, &size) != 0) return error.GpuBackend;
            const na: usize = @intCast(req.n_accounts);
            const np: usize = na + @as(usize, @intCast(req.n_slots));
            const A = struct {
                fn get(a: Allocator, comptime T: type, n: usize) Error![]T {
                    return a.alloc(T, n + 1) catch return error.OutOfMemory;
                }
            };
            const nodes = try A.get(arena, u8, @intCast(size.nodes_bytes));
            const node_off = try A.get(arena, u64, @intCast(size.n_nodes));
            const node_index = try A.get(arena, u64, @intCast(size.n_refs));
            const proof_first = try A.get(arena, u64, np);
            const roots32 = try A.get(arena, u8, 32 * np);
            const status = try A.get(arena, u8, np);
            const nonce = try A.get(arena, u64, na);
            const balance32 = try A.get(arena, u8, 32 * na);
            const storage_root32 = try A.get(arena, u8, 32 * na);
            const code_hash32 = try A.get(arena, u8, 32 * na);
            const slot_vals32 = try A.get(arena, u8, 32 * (np - na));
            var out = c.phant_gpu_proofs{ .nodes = nodes.ptr, .node_off = node_off.ptr, .node_index = node_index.ptr, .proof_first = proof_first.ptr,
                .roots32 = roots32.ptr, .status = status.ptr, .nonce = nonce.ptr, .balance32 = balance32.ptr, .storage_root32 = storage_root32.ptr,
                .code_hash32 = code_hash32.ptr, .slot_vals32 = slot_vals32.ptr };
            if (c.phant_gpu_resident_state_prove_copy(self.s, &out) != 0) return error.GpuBackend;
            return .{ .nodes = nodes[0..@intCast(size.nodes_bytes)], .node_off = node_off, .node_index = node_index[0..@intCast(size.n_refs)],
                .proof_first = proof_first, .roots32 = roots32[0 .. 32 * np], .status = status[0..np], .nonce = nonce[0..na],
                .balance32 = balance32[0 .. 32 * na], .storage_root32 = storage_root32[0 .. 32 * na], .code_hash32 = code_hash32[0 .. 32 * na],
                .slot_vals32 = slot_vals32[0 .. 32 * (np - na)] };
        }
        /// Account and slot values (eth_getBalance, eth_getTransactionCount, eth_getStorageAt, the codeHash behind
        /// eth_getCode) of the state as it is now (back = 0) or as it was `back` applies ago, read without changing it; the
        /// request is prove's, repeated keys allowed.  Also returns the root the values belong to.  Every array is allocated
        /// in `arena`.  Not compiled: the build has no Zig toolchain.
        pub fn read(self: *ResidentState, arena: Allocator, req: *const c.phant_gpu_proof_request, back: u32) Error!struct {
            root: [32]u8,
            account_status: []u8,
            nonce: []u64,
            balance32: []u8,
            storage_root32: []u8,
            code_hash32: []u8,
            slot_status: []u8,
            slot_vals32: []u8,
        } {
            const na: usize = @intCast(req.n_accounts);
            const ms: usize = @intCast(req.n_slots);
            const A = struct {
                fn get(a: Allocator, comptime T: type, n: usize) Error![]T {
                    return a.alloc(T, n + 1) catch return error.OutOfMemory;
                }
            };
            const account_status = try A.get(arena, u8, na);
            const nonce = try A.get(arena, u64, na);
            const balance32 = try A.get(arena, u8, 32 * na);
            const storage_root32 = try A.get(arena, u8, 32 * na);
            const code_hash32 = try A.get(arena, u8, 32 * na);
            const slot_status = try A.get(arena, u8, ms);
            const slot_vals32 = try A.get(arena, u8, 32 * ms);
            var out = c.phant_gpu_state_read_values{ .account_status = account_status.ptr, .nonce = nonce.ptr, .balance32 = balance32.ptr,
                .storage_root32 = storage_root32.ptr, .code_hash32 = code_hash32.ptr, .slot_status = slot_status.ptr, .slot_vals32 = slot_vals32.ptr };
            var root: [32]u8 = undefined;
            if (c.phant_gpu_resident_state_read(self.s, req, back, &out, &root) != 0) return error.GpuBackend;
            return .{ .root = root, .account_status = account_status[0..na], .nonce = nonce[0..na], .balance32 = balance32[0 .. 32 * na],
                .storage_root32 = storage_root32[0 .. 32 * na], .code_hash32 = code_hash32[0 .. 32 * na], .slot_status = slot_status[0..ms],
                .slot_vals32 = slot_vals32[0 .. 32 * ms] };
        }
        /// Account and storage ranges (debug_accountRange, debug_storageRangeAt, snap's GetAccountRange / GetStorageRanges
        /// without proofs) of the state as it is now (back = 0) or as it was `back` applies ago, read without changing it.
        /// Range r's entries are [account_first[r], account_first[r + 1]) (slot_first for storage ranges); `more` says
        /// whether the range holds further keys.  Entry arrays are sized by the sum of the request's max values; every array
        /// is allocated in `arena`.  Not compiled: the build has no Zig toolchain.
        pub fn range(self: *ResidentState, arena: Allocator, req: *const c.phant_gpu_range_request, back: u32) Error!struct {
            root: [32]u8,
            account_first: []u64,
            account_more: []u8,
            account_keys32: []u8,
            nonce: []u64,
            balance32: []u8,
            storage_root32: []u8,
            code_hash32: []u8,
            slot_first: []u64,
            slot_more: []u8,
            slot_keys32: []u8,
            slot_vals32: []u8,
        } {
            const n: usize = @intCast(req.n_account_ranges);
            const m: usize = @intCast(req.n_storage_ranges);
            var ea: usize = 0;
            var es: usize = 0;
            for (0..n) |r| ea += req.account_max[r];
            for (0..m) |r| es += req.storage_max[r];
            const A = struct {
                fn get(a: Allocator, comptime T: type, len: usize) Error![]T {
                    return a.alloc(T, len + 1) catch return error.OutOfMemory;
                }
            };
            const account_first = try A.get(arena, u64, n + 1);
            const account_more = try A.get(arena, u8, n);
            const account_keys32 = try A.get(arena, u8, 32 * ea);
            const nonce = try A.get(arena, u64, ea);
            const balance32 = try A.get(arena, u8, 32 * ea);
            const storage_root32 = try A.get(arena, u8, 32 * ea);
            const code_hash32 = try A.get(arena, u8, 32 * ea);
            const slot_first = try A.get(arena, u64, m + 1);
            const slot_more = try A.get(arena, u8, m);
            const slot_keys32 = try A.get(arena, u8, 32 * es);
            const slot_vals32 = try A.get(arena, u8, 32 * es);
            var out = c.phant_gpu_range_values{ .account_first = account_first.ptr, .account_more = account_more.ptr,
                .account_keys32 = account_keys32.ptr, .nonce = nonce.ptr, .balance32 = balance32.ptr, .storage_root32 = storage_root32.ptr,
                .code_hash32 = code_hash32.ptr, .slot_first = slot_first.ptr, .slot_more = slot_more.ptr, .slot_keys32 = slot_keys32.ptr,
                .slot_vals32 = slot_vals32.ptr };
            var root: [32]u8 = undefined;
            if (c.phant_gpu_resident_state_range(self.s, req, back, &out, &root) != 0) return error.GpuBackend;
            const na: usize = @intCast(account_first[n]);
            const ms: usize = @intCast(slot_first[m]);
            return .{ .root = root, .account_first = account_first[0 .. n + 1], .account_more = account_more[0..n],
                .account_keys32 = account_keys32[0 .. 32 * na], .nonce = nonce[0..na], .balance32 = balance32[0 .. 32 * na],
                .storage_root32 = storage_root32[0 .. 32 * na], .code_hash32 = code_hash32[0 .. 32 * na], .slot_first = slot_first[0 .. m + 1],
                .slot_more = slot_more[0..m], .slot_keys32 = slot_keys32[0 .. 32 * ms], .slot_vals32 = slot_vals32[0 .. 32 * ms] };
        }
        /// Keep contract code on the device beside the state, by keccak(code): code i = codes[code_off[i] .. code_off[i + 1]).
        /// A code already held is stored once, the empty code never.  hashes32 (n * 32 bytes, or null) gets the hashes in
        /// order.  Not compiled: the build has no Zig toolchain.
        pub fn putCodes(self: *ResidentState, codes: []const u8, code_off: []const u64, hashes32: ?[]u8) Error!void {
            const n = code_off.len - 1;
            if (c.phant_gpu_resident_state_put_codes(self.s, codes.ptr, code_off.ptr, n, if (hashes32) |h| h.ptr else null) != 0)
                return error.GpuBackend;
        }
        /// The codes behind n hashes (eth_getCode after read, snap's GetByteCodes): status (1 held, 2 not held) and CSR
        /// offsets into the returned bytes, all allocated in `arena`.  Two calls: the sizes, then the bytes.
        pub fn codes(self: *ResidentState, arena: Allocator, hashes32: []const u8) Error!struct { status: []u8, code_off: []u64, codes: []u8 } {
            const n = hashes32.len / 32;
            const status = arena.alloc(u8, n + 1) catch return error.OutOfMemory;
            const code_off = arena.alloc(u64, n + 1) catch return error.OutOfMemory;
            if (c.phant_gpu_resident_state_codes(self.s, hashes32.ptr, n, status.ptr, code_off.ptr, null, 0) != 0) return error.GpuBackend;
            const total: usize = @intCast(code_off[n]);
            const bytes = arena.alloc(u8, total + 1) catch return error.OutOfMemory;
            if (total != 0 and c.phant_gpu_resident_state_codes(self.s, hashes32.ptr, n, status.ptr, code_off.ptr, bytes.ptr, total) != 0)
                return error.GpuBackend;
            return .{ .status = status[0..n], .code_off = code_off, .codes = bytes[0..total] };
        }
        /// The node at each requested nibble path of the account trie or of a named storage trie (snap's GetTrieNodes) under
        /// the current root: status (1 served, 2 no node) and CSR offsets into the returned node bytes, in request order,
        /// all allocated in `arena`.  Not compiled: the build has no Zig toolchain.
        pub fn trieNodes(self: *ResidentState, arena: Allocator, req: *const c.phant_gpu_trie_node_request) Error!struct {
            status: []u8,
            node_off: []u64,
            nodes: []u8,
        } {
            const n: usize = @intCast(req.n_paths);
            var size: c.phant_gpu_witness_size = undefined;
            if (c.phant_gpu_resident_state_trie_nodes(self.s, req, &size) != 0) return error.GpuBackend;
            const total: usize = @intCast(size.nodes_bytes);
            const status = arena.alloc(u8, n + 1) catch return error.OutOfMemory;
            const node_off = arena.alloc(u64, n + 1) catch return error.OutOfMemory;
            const nodes = arena.alloc(u8, total + 1) catch return error.OutOfMemory;
            var out = c.phant_gpu_trie_nodes{ .status = status.ptr, .node_off = node_off.ptr, .nodes = nodes.ptr };
            if (c.phant_gpu_resident_state_trie_nodes_copy(self.s, &out) != 0) return error.GpuBackend;
            return .{ .status = status[0..n], .node_off = node_off, .nodes = nodes[0..total] };
        }
        /// The answers of snap GetAccountRange and GetStorageRanges requests under the current root, with byte budgets, slim
        /// account bodies and boundary proof lists (include/phant_gpu.h, DESIGN.md §4.3m): every array of
        /// phant_gpu_snap_ranges allocated in `arena` and filled.  Serve a pivot through fork().  Not compiled: the build has
        /// no Zig toolchain.
        pub fn snapRanges(self: *ResidentState, arena: Allocator, req: *const c.phant_gpu_snap_request) Error!struct {
            size: c.phant_gpu_snap_size,
            out: c.phant_gpu_snap_ranges,
        } {
            var size: c.phant_gpu_snap_size = undefined;
            if (c.phant_gpu_resident_state_snap_ranges(self.s, req, &size) != 0) return error.GpuBackend;
            const n: usize = @intCast(req.n_account_requests);
            const m: usize = @intCast(req.n_storage_requests);
            const u64s = struct {
                fn take(a: Allocator, k: u64) Error![*]u64 {
                    return (a.alloc(u64, @as(usize, @intCast(k)) + 1) catch return error.OutOfMemory).ptr;
                }
                fn bytes(a: Allocator, k: u64) Error![*]u8 {
                    return (a.alloc(u8, @as(usize, @intCast(k)) + 1) catch return error.OutOfMemory).ptr;
                }
            };
            var out = c.phant_gpu_snap_ranges{
                .account_first = try u64s.take(arena, n + 1),
                .account_keys32 = try u64s.bytes(arena, 32 * size.n_accounts),
                .account_body_off = try u64s.take(arena, size.n_accounts + 1),
                .account_bodies = try u64s.bytes(arena, size.account_bytes),
                .served_first = try u64s.take(arena, m + 1),
                .slot_first = try u64s.take(arena, size.n_served + 1),
                .slot_keys32 = try u64s.bytes(arena, 32 * size.n_slots),
                .slot_body_off = try u64s.take(arena, size.n_slots + 1),
                .slot_bodies = try u64s.bytes(arena, size.slot_bytes),
                .proof_first = try u64s.take(arena, n + m + 1),
                .node_index = try u64s.take(arena, size.n_refs),
                .nodes = try u64s.bytes(arena, size.nodes_bytes),
                .node_off = try u64s.take(arena, size.n_nodes + 1),
            };
            if (c.phant_gpu_resident_state_snap_ranges_copy(self.s, &out) != 0) return error.GpuBackend;
            return .{ .size = size, .out = out };
        }
        /// Drop the held codes no account names now or at any root the journal reaches.
        pub fn pruneCodes(self: *ResidentState) Error!void {
            if (c.phant_gpu_resident_state_prune_codes(self.s) != 0) return error.GpuBackend;
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
