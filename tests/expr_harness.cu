// expr_harness.cu -- the fused expression path's host compiler (expr_compile in csrc/k_expr.cu) as a host program, driven by
// tests/test_expr_programs.py.  expr_compile is hidden in the library (-fvisibility=hidden), so this file includes k_expr.cu itself;
// nvcc compiles the kernels too, but nothing here launches one, so the program runs without a GPU.
//
// stdin: one DAG per line, "n_inputs n_nodes op a b op a b ..." (the C ABI's node ops: 0..6 binary, 100 + unop unary, and b == a
// for a unary node, as bdf_expr_check passes them).
// stdout: one line per DAG, "code n_ins n_slots op src op src ..." (the ExprProg when code == 0, "code 0 0" otherwise).
// With the argument "constants": the compiler's limits and tile sizes, one "name value" per line.
#include <cstdio>
#include <cstdlib>

#include "k_expr.cu"

int main(int argc, char** argv) {
    using namespace bdf;
    if (argc > 1 && argv[1][0] == 'c') {
        printf("kExprMaxInputs %d\nkExprMaxNodes %d\nkExprMaxIns %d\nkExprMaxTemps %d\nkExprUnroll %d\nkBulkU %d\nkThreads %d\n"
               "expr_tile_elems %d\nXI_BIN %d\nXI_RBIN %d\nXI_LOAD %d\nXI_STORE %d\nXI_UN %d\nkOperandAcc %d\n",
               kExprMaxInputs, kExprMaxNodes, kExprMaxIns, kExprMaxTemps, kExprUnroll, kBulkU, kThreads, expr_tile_elems(),
               (int)XI_BIN, (int)XI_RBIN, (int)XI_LOAD, (int)XI_STORE, (int)XI_UN, kOperandAcc);
        return 0;
    }
    static char line[1 << 12];
    int dt[kExprMaxInputs];
    for (int i = 0; i < kExprMaxInputs; i++) dt[i] = T_F64;
    while (fgets(line, sizeof(line), stdin)) {
        char* p = line;
        char* q;
        const int ni = (int)strtol(p, &q, 10);
        if (q == p) continue;
        p = q;
        const int nn = (int)strtol(p, &p, 10);
        if (ni < 1 || ni > kExprMaxInputs || nn < 1 || nn > kExprMaxNodes) { fprintf(stderr, "bad DAG: %s", line); return 2; }
        int op[kExprMaxNodes], a[kExprMaxNodes], b[kExprMaxNodes];
        for (int k = 0; k < nn; k++) {
            op[k] = (int)strtol(p, &p, 10); a[k] = (int)strtol(p, &p, 10); b[k] = (int)strtol(p, &p, 10);
            if (a[k] < 0 || a[k] >= ni + k || b[k] < 0 || b[k] >= ni + k) { fprintf(stderr, "forward reference: %s", line); return 2; }
        }
        ExprProg prog;
        const int code = expr_compile(ni, dt, nn, op, a, b, &prog);
        if (code != 0) { printf("%d 0 0\n", code); continue; }
        printf("0 %d %d", prog.n_ins, prog.n_slots);
        for (int k = 0; k < prog.n_ins; k++) printf(" %d %d", (int)prog.op[k], (int)prog.src[k]);
        putchar('\n');
    }
    return 0;
}
