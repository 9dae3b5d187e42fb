// cuba_structure.h -- host-side construction of every index structure of the LM path from the flat
// (iP,iL) edge list.  Pure C++ (no CUDA) so the not-gpu tests can exercise it through
// cuba_debug_build_structure_host().
//
// What it replaces in the reference (paths relative to the reference checkout):
//   gpu::buildHplStructure            src/cuda_block_solver.cu:1158-1173   (Hpl CSC, edge2Hpl)
//   HschurSparseBlockMatrix::constructFromVertices  src/sparse_block_matrix.cpp:55-133 (Hsc upper BSR)
//   gpu::findHschureMulBlockIndices   cu:979-1000,1175-1190                 (block-product list)
// plus what is new here: the canonical (iL,iP) edge order, landmark tiles, the pose-major edge copy,
// the destination-sorted product list and the symmetric-full BSR used by the PCG.
#pragma once

#include <cstdint>
#include <vector>

namespace cuba_b200 {

struct Structure {
	// sizes
	int Pall = 0, numP = 0, Lall = 0, numL = 0, E2 = 0, E3 = 0, E = 0;
	int nhpl = 0;          // global number of Hpl blocks (free-free edges)
	int nblk = 0;          // upper-triangular Hsc blocks
	long long nmul = 0;    // global number of block products
	int nfull = 0;         // blocks of the symmetric-full BSR
	// landmark shard owned by this rank: landmarks [lmBeg, lmEnd)
	int lmBeg = 0, lmEnd = 0;
	int eLocal = 0;        // edges of the shard
	int hplBase = 0;       // first global Hpl index of the shard
	int nhplLocal = 0;
	long long nmulLocal = 0;
	bool repeatedPairs = false;   // some free pose observes some free landmark through more than one edge

	// global structures (bit-exact contract with the reference)
	std::vector<int> hplColPtr;   // [numL+1]
	std::vector<int> hplRowInd;   // [nhpl]
	std::vector<int> edge2Hpl;    // [E] user edge id -> Hpl block (-1 when an end is fixed)
	std::vector<int> hscRowPtr;   // [numP+1] upper BSR
	std::vector<int> hscColInd;   // [nblk]

	// landmark-major edge stream of the shard (sorted by (iL,iP,edge id))
	std::vector<int> order;       // [eLocal] user edge id of each stream slot
	std::vector<int> e_ip;        // bit31 = stereo
	std::vector<int> e_il;
	std::vector<int> e_hpl;       // LOCAL Hpl index, or -1-rank (rank among the shard's free-free edges) if no block
	std::vector<int> lmPtr;       // [Lall+1] stream offsets; landmarks outside the shard have empty runs
	std::vector<int> tileLm;      // [ntiles+1] first landmark of each tile
	std::vector<int> hplLm;       // [nhplLocal] landmark of each local Hpl block

	// pose-major stream of the shard (free poses only), sorted by (iP,iL)
	std::vector<int> posePtr;     // [numP+1]
	std::vector<int> p_src;       // [npose_edges] landmark-major slot each entry was copied from
	std::vector<int> p_il;        // bit31 = stereo

	// destination-sorted product list of the shard's landmarks
	std::vector<int> blkRow, blkCol;   // [nblk]
	std::vector<int> prodPtr;          // [nblk+1]
	std::vector<int> prodI, prodJ;     // [nmulLocal] LOCAL Hpl indices, row(prodI) <= row(prodJ); on a diagonal destination
	                                   // every ordered pair of the pose's blocks of one landmark (both (i, j) and (j, i))

	// symmetric-full BSR
	std::vector<int> fRowPtr;     // [numP+1]
	std::vector<int> fColInd;     // [nfull]
	std::vector<int> u2f, u2fT;   // [nblk] upper block -> full position of (a,b) and of (b,a)
};

// idx2/idx3: (iP,iL) pairs.  rank/world select the landmark shard (world==1: everything).
// Returns false and fills err on inconsistent input.
bool build_structure(int Pall, int numP, int Lall, int numL, int E2, const int32_t* idx2, int E3, const int32_t* idx3,
	int rank, int world, int tileEdges, Structure& S, const char** err);

// ---- host side of the PCG setup (pure C++, tested on the CPU through cuba_debug_pcg_partition) --------------------
// (Engine::setup_pcg2 in cuba_engine.cu calls these functions: one implementation for the engine and for the CPU tests.)
// Row partition of the reduced pose system over G persistent CTAs: contiguous row ranges balanced by block count, the sorted
// list of block columns every CTA needs, and the position of each block's column in that list (diagonal blocks: -1-pos).
struct PcgPartition {
	int G = 0;
	std::vector<int> rows;     // [G+1]
	std::vector<int> nptr;     // [G+1] offsets into ncol
	std::vector<int> ncol;     // needed columns per CTA, ascending
	std::vector<int> local;    // [nfull]
	int needMax = 0, blkMax = 0, maxRows = 0;
};
// contiguous row ranges balanced by block count; with maxRows > 0 no range is longer than maxRows (balanced as far as that allows)
void build_pcg_partition(int numP, int nfull, const std::vector<int>& fRowPtr, const std::vector<int>& fColInd, int G, PcgPartition& P,
	int maxRows = 0);

// Coarse level of the two-level PCG: aggregates = groups of gs consecutive CTAs (at most maxAgg of them), the aggregates every
// CTA needs, and -- build_coarse_lists -- the fine blocks of every coarse block of the lower triangle in ascending order.
// With apc > 1 aggregates per CTA instead (gs = 1, A = apc G): the CTA's rows cut into apc contiguous groups balanced by row count,
// aggregate c apc + j = group j of CTA c; A = 0 when some CTA has fewer than apc rows.
struct CoarsePartition {
	int gs = 1, apc = 1, A = 0, maxNeedAgg = 1;
	std::vector<int> aggRow;   // [A+1] first row of every aggregate
	std::vector<int> rowAgg;   // [numP]
	std::vector<int> naPtr;    // [G+1]
	std::vector<int> naList;   // aggregates per CTA, ascending
	std::vector<int> needAgg;  // per need entry: position of its aggregate in the CTA's list
	std::vector<int> rowOf;    // [nfull] row of every block
	std::vector<int> cbPtr;    // [A(A+1)/2 + 1]
	std::vector<int> cbList;   // fine blocks of coarse block (ib >= jb) at index ib (ib+1)/2 + jb
};
void build_coarse_partition(int numP, const PcgPartition& P, int maxAgg, CoarsePartition& C, int apc = 1);
void build_coarse_lists(int numP, int nfull, const std::vector<int>& fRowPtr, const std::vector<int>& fColInd, CoarsePartition& C);
// invariants of both (nullptr when everything holds)
const char* check_pcg_partition(int numP, int nfull, const std::vector<int>& fRowPtr, const std::vector<int>& fColInd,
	const PcgPartition& P, const CoarsePartition& C);

// Plan of the row-distributed two-level PCG (k_pcg5): rows cut into world x G contiguous ranges ("virtual CTAs"), G per GPU;
// aggregates = groups of gs consecutive virtual CTAs with gs | G, so that no aggregate straddles two ranks; rowPeers[j] = bit
// mask of the ranks (other than the owner) whose CTAs need row j's w entries.  ok == false: the system is too small / the row
// ranges too long for the kernel (the engine then keeps the older kernels).  apc > 1 (one GPU only): apc aggregates per CTA.
struct Pcg5Plan {
	bool ok = false;
	int world = 1, G = 0, gs = 1, A = 0, apc = 1;
	PcgPartition P;
	CoarsePartition C;
	std::vector<unsigned char> rowPeers;
};
// `same`: a partition of the same system the caller already has (k_pcg3's); copied instead of rebuilt when its CTA count fits.
void build_pcg5_plan(int numP, int nfull, const std::vector<int>& fRowPtr, const std::vector<int>& fColInd, int world, int numSMs, int maxAgg,
	int maxRowsPerCta, Pcg5Plan& plan, const PcgPartition* same = nullptr, int apc = 1);
// The direct solver (cuba_dense_chol.cuh): the block of the symmetric-full BSR behind every block of the packed lower block
// triangle of S -- block (i >= j) at i (i+1)/2 + j, -1 where S has none.  Built once per structure.
void build_dense_block_map(int numP, const std::vector<int>& fRowPtr, const std::vector<int>& fColInd, std::vector<int>& map);

// invariants of a plan (nullptr when everything holds)
const char* check_pcg5_plan(int numP, int nfull, const std::vector<int>& fRowPtr, const std::vector<int>& fColInd, const Pcg5Plan& plan);

}  // namespace cuba_b200
