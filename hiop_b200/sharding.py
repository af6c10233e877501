"""Layouts of the multi-rank paths.

Column (n) partition of the quasi-Newton KKT path over ranks/GPUs -- the reference's MPI layout
(src/Optimization/hiopHessianLowRank.hpp:88-89, col_part in src/LinAlg/hiopVectorPar.cpp:78-87): every n-vector and the
columns of J, S_t, Y_t are split, every m- and l-sized object is replicated, and each reduction the reference does with
MPI_Allreduce becomes one sum all-reduce (NCCL inside libhiopb200.so, see hb_comm_init)."""
from __future__ import annotations


# block size of the distributed dense factorization (hb_symdense_dist.cu; = hb_big_factor's)
DIST_BLOCK = 128


def block_rows(N: int, world: int, rank: int) -> list[tuple[int, int]]:
    """[begin, end) of the global rows of each block row `rank` owns in the 1-D block-cyclic layout of hb_symdense_dist, in the order
    they are stacked in its local storage: block row k (rows k*128 .. min(N, k*128+128)) belongs to rank k mod world."""
    nblk = (N + DIST_BLOCK - 1) // DIST_BLOCK
    return [(k * DIST_BLOCK, min(N, (k + 1) * DIST_BLOCK)) for k in range(rank, nblk, world)]


def column_range(n: int, world: int, rank: int) -> tuple[int, int]:
    """[begin, end) of the columns owned by `rank`; the first n % world ranks own one extra column."""
    base, rem = divmod(n, world)
    begin = rank * base + min(rank, rem)
    return begin, begin + base + (1 if rank < rem else 0)


# the sum all-reduces of one condensed KKT system, in order, with their payload in doubles (m constraints, l secant pairs)
def reductions_per_system(m: int, l: int) -> list[tuple[str, int]]:
    return [
        ("S S^T (once per secant update; hiopHessianLowRank.cpp:459 carries it inside the 3 l^2 message)", l * l),
        ("C_aug = [J;S;Y] DhInv [J;S;Y]^T: W, S1, Y1 and V's blocks in one message (hiopHessianLowRank.cpp:459,590,591)", (m + 2 * l) ** 2),
        ("[sigma S (DhInv r); Y (DhInv r)] of each hiopHessianLowRank::solve (hiopHessianLowRank.cpp:515,520)", 2 * l),
        ("J dx_tmp (hiopMatrixDenseRowMajor.cpp:487, beta applied on rank 0 only :464-467)", m),
        ("second hiopHessianLowRank::solve", 2 * l),
    ]


# compound (12-block) vectors of the outer refinement: which blocks are sharded along n and which are replicated on every rank
N_BLOCKS = ("x", "sxl", "sxu", "zl", "zu")
M_BLOCKS = ("d", "yc", "yd", "sdl", "sdu", "vl", "vu")


def compound_reduction_contribution(rank: int, blocks: dict, op):
    """What one rank feeds into the single all-reduce of a compound-vector reduction (dot, squared 2-norm, ...): its shard of the
    n-sized blocks always, the replicated m-sized blocks only on rank 0 -- the rule hb_krylov.cu implements by shortening the
    reduction length on ranks != 0 (hiopVectorCompoundPD reduces each block in its own communicator instead,
    src/LinAlg/hiopVectorCompoundPD.cpp:438-461). `op(block_name, array) -> float` is the local reduction of one block."""
    total = sum(op(k, blocks[k]) for k in N_BLOCKS)
    if rank == 0:
        total += sum(op(k, blocks[k]) for k in M_BLOCKS)
    return total
