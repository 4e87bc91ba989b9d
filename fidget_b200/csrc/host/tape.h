// Host-side tape front end for the H100 backend.
//
// This is the part of Fidget that "stays on the host" for every backend
// (SURVEY.md §1, "TAPE / COMPILER"): a hash-consed expression context with
// the `.vm` text loader, the SSA flattening, the single-pass register
// allocator and the packed bytecode writer.  In a Rust integration these
// roles are played by the reference's own fidget-core / fidget-bytecode
// crates; this C++ mirror exists so that the CUDA backend can be driven (from
// C++ or Python) without a Rust toolchain, and produces *the same* tapes:
//
//   Context / from_text   <-> fidget-core/src/context/mod.rs:49-322,878-941
//   SsaTape::build        <-> fidget-core/src/compiler/ssa_tape.rs:39-261
//   RegAlloc              <-> fidget-core/src/compiler/alloc.rs:13-708
//   RegTape / repack_map  <-> fidget-core/src/compiler/reg_tape.rs:9-113
//   bytecode()            <-> fidget-bytecode/src/lib.rs:203-332
//
// Nothing in here touches the GPU.
#pragma once
#include <cstdint>
#include <string>
#include <unordered_map>
#include <vector>

namespace fhost {

// Opcode numbering == fidget_bytecode::BytecodeOp declaration order
// (fidget-bytecode/src/lib.rs:69-104); this is the wire format.
enum Opcode : uint8_t {
    OP_OUTPUT = 0, OP_INPUT, OP_COPY, OP_NEG, OP_ABS, OP_RECIP, OP_SQRT,
    OP_SQUARE, OP_FLOOR, OP_CEIL, OP_ROUND, OP_NOT, OP_RAND, OP_SIN, OP_COS,
    OP_TAN, OP_ASIN, OP_ACOS, OP_ATAN, OP_EXP, OP_LN, OP_ADD, OP_SUB, OP_MUL,
    OP_DIV, OP_ATAN2, OP_COMPARE, OP_MIX, OP_MOD, OP_MIN, OP_MAX, OP_AND,
    OP_OR, OP_MEM, OP_COUNT
};
const char* opcode_name(uint8_t op);
inline bool is_unary(uint8_t op) { return op >= OP_NEG && op <= OP_LN; }
inline bool is_binary(uint8_t op) { return op >= OP_ADD && op <= OP_OR; }
inline bool is_choice(uint8_t op) { return op >= OP_MIN && op <= OP_OR; }

// Which operand of a binary clause is an immediate.
enum Form : uint8_t { F_RR = 0, F_RI = 1, F_IR = 2 };

// One clause of a tape.  The same struct describes SSA clauses (out/a/b are
// SSA indices) and register clauses (out/a/b are slots; slots >= N are
// memory).  Layout by opcode:
//   OUTPUT : a = source,  idx = output index
//   INPUT  : out = dest,  idx = variable index
//   COPY   : out, a (F_RR) or imm (F_RI: "CopyImm")
//   unary  : out, a
//   binary : out, a, b / imm according to `form`
//            (F_RI: a OP imm,  F_IR: imm OP a -- the register is always `a`)
//   MEM    : load  = out <- mem[idx]  (form F_RI)
//            store = mem[idx] <- a    (form F_IR)
struct Clause {
    uint8_t op = 0;
    uint8_t form = F_RR;
    uint32_t out = 0, a = 0, b = 0;
    uint32_t idx = 0;
    float imm = 0.f;
    bool operator==(const Clause& o) const;
};
std::string to_string(const Clause& c);

////////////////////////////////////////////////////////////////////////////
// Variables (fidget-core/src/var/mod.rs:32,105-148)
struct Var {
    enum Kind : uint8_t { X, Y, Z, V } kind = X;
    uint64_t id = 0;  // only for V
    bool operator==(const Var& o) const { return kind == o.kind && (kind != V || id == o.id); }
};

// var -> input slot, assigned in discovery order
struct VarMap {
    std::vector<Var> order;  // index -> var
    int get(const Var& v) const;
    void insert(const Var& v);
    size_t size() const { return order.size(); }
};

////////////////////////////////////////////////////////////////////////////
// Expression context with deduplication and constant folding
using Node = uint32_t;
class Context {
public:
    enum Kind : uint8_t { K_CONST, K_VAR, K_UNARY, K_BINARY };
    struct Op {
        Kind kind;
        uint8_t op;   // Opcode for unary/binary
        Node a, b;
        float value;  // K_CONST
        Var var;      // K_VAR
    };
    Node constant(float f);
    Node var(Var v);
    Node x() { return var(Var{Var::X, 0}); }
    Node y() { return var(Var{Var::Y, 0}); }
    Node z() { return var(Var{Var::Z, 0}); }
    Node fresh_var();  // Var::new() equivalent (unique id)

    Node unary(uint8_t op, Node a);     // generic, with folding
    Node add(Node a, Node b);
    Node sub(Node a, Node b);
    Node mul(Node a, Node b);
    Node div(Node a, Node b);
    Node min(Node a, Node b);
    Node max(Node a, Node b);
    Node and_(Node a, Node b);
    Node or_(Node a, Node b);
    Node atan2(Node y, Node x);
    Node compare(Node a, Node b);
    Node mix(Node a, Node b);
    Node modulo(Node a, Node b);
    Node neg(Node a) { return unary(OP_NEG, a); }
    Node square(Node a) { return unary(OP_SQUARE, a); }
    Node sqrt(Node a) { return unary(OP_SQRT, a); }
    Node abs(Node a) { return unary(OP_ABS, a); }
    Node sin(Node a) { return unary(OP_SIN, a); }
    Node cos(Node a) { return unary(OP_COS, a); }
    Node not_(Node a) { return unary(OP_NOT, a); }
    Node recip(Node a) { return unary(OP_RECIP, a); }

    // Parses the `.vm` text format; returns the root (last line).  Throws
    // std::runtime_error on unknown opcodes / names / empty input.
    Node from_text(const std::string& text);

    const Op& get(Node n) const { return ops_[n]; }
    size_t size() const { return ops_.size(); }
    bool is_const(Node n, float* v = nullptr) const;

    // Scalar point evaluation of the graph (used to fold constants and by
    // tests); `vars` indexed by position in `vm`.
    static float eval_unary(uint8_t op, float a);
    static float eval_binary(uint8_t op, float a, float b);

private:
    Node intern(const Op& op);
    Node binary(uint8_t op, Node a, Node b);
    Node binary_commutative(uint8_t op, Node a, Node b);
    std::vector<Op> ops_;
    std::unordered_map<std::string, Node> dedup_;
    uint64_t next_var_ = 0;
};

////////////////////////////////////////////////////////////////////////////
// SSA tape: clauses stored ROOT FIRST (reverse evaluation order)
struct SsaTape {
    std::vector<Clause> tape;
    uint32_t choice_count = 0;
    uint32_t output_count = 0;
    static SsaTape build(const Context& ctx, const std::vector<Node>& roots, VarMap* vars);
};

// Register tape: clauses stored ROOT FIRST; slots 0..N are registers, N.. memory
struct RegTape {
    std::vector<Clause> tape;
    uint32_t slot_count = 0;
    size_t len() const { return tape.size(); }
};

// Single-pass allocator; fed SSA clauses root first.
class RegAlloc {
public:
    RegAlloc(uint32_t n_regs, size_t ssa_len);
    void op(const Clause& c);
    RegTape finalize();

private:
    static constexpr uint32_t UNASSIGNED = 0xFFFFFFFFu;
    struct Lru {
        std::vector<uint8_t> prev, next;
        uint8_t head = 0;
        explicit Lru(uint32_t n);
        void remove(uint8_t i);
        void insert_before(uint8_t i, uint8_t nx);
        void poke(uint8_t i);
        uint8_t pop();
    };
    enum AKind { A_REG, A_MEM, A_NONE };
    struct Alloc { AKind k; uint32_t v; };

    uint32_t N;
    std::vector<uint32_t> allocations;  // ssa index -> slot | UNASSIGNED
    std::vector<uint32_t> registers;    // register -> ssa index | UNASSIGNED
    Lru lru;
    std::vector<uint8_t> spare_registers;
    std::vector<uint32_t> spare_memory;
    RegTape out;

    uint32_t get_memory();
    Alloc get_allocation(uint32_t n);
    uint8_t get_register();
    void rebind_register(uint32_t n, uint8_t reg);
    void bind_register(uint32_t n, uint8_t reg);
    void release_reg(uint8_t reg);
    void push_store(uint8_t reg, uint32_t mem);
    uint8_t get_out_reg(uint32_t o);
    void op_one_arg(const Clause& c);
    void op_two_args(const Clause& c);
    void op_out_only(const Clause& c);
    void op_output(const Clause& c);
    void emit(Clause c, uint32_t o, uint32_t a, uint32_t b);
};

RegTape allocate_registers(const SsaTape& ssa, uint32_t n_regs);

// Both tape forms + the variable map (fidget-core/src/vm/data.rs:65-86)
struct TapeData {
    SsaTape ssa;
    RegTape asm_;
    VarMap vars;
    uint32_t n_regs = 255;
    static TapeData build(const Context& ctx, const std::vector<Node>& roots, uint32_t n_regs = 255);
    size_t len() const { return asm_.len(); }
};

// Packed wire format
struct Bytecode {
    std::vector<uint32_t> words;  // incl. start/end markers
    uint8_t reg_count = 0;
    uint32_t mem_count = 0;
};
// `repack` applies the frequency repacking of Bytecode::new; throws if a
// packed register would be 255.
Bytecode make_bytecode(const RegTape& t, uint32_t n_regs, bool repack = true);

}  // namespace fhost
