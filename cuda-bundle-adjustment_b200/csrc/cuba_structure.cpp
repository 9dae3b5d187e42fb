// cuba_structure.cpp -- see cuba_structure.h
#include "cuba_structure.h"

#include <algorithm>

namespace cuba_b200 {

bool build_structure(int Pall, int numP, int Lall, int numL, int E2, const int32_t* idx2, int E3, const int32_t* idx3,
	int rank, int world, int tileEdges, Structure& S, const char** err)
{
	S = Structure();
	if (Pall < 0 || Lall < 0 || numP < 0 || numL < 0 || numP > Pall || numL > Lall || E2 < 0 || E3 < 0 || world < 1 || rank < 0 ||
		rank >= world || tileEdges < 1) {
		*err = "build_structure: invalid sizes";
		return false;
	}
	const int E = E2 + E3;
	S.Pall = Pall; S.numP = numP; S.Lall = Lall; S.numL = numL; S.E2 = E2; S.E3 = E3; S.E = E;
	auto IP = [&](int u) { return u < E2 ? idx2[2 * (size_t)u] : idx3[2 * (size_t)(u - E2)]; };
	auto IL = [&](int u) { return u < E2 ? idx2[2 * (size_t)u + 1] : idx3[2 * (size_t)(u - E2) + 1]; };
	for (int u = 0; u < E; u++) {
		const int ip = IP(u), il = IL(u);
		if (ip < 0 || ip >= Pall || il < 0 || il >= Lall) { *err = "build_structure: edge index out of range"; return false; }
		if (ip >= numP && il >= numL) { *err = "build_structure: edge with both ends fixed"; return false; }
	}

	// 1. canonical order: stable counting sort by iP, then by iL  ->  sorted by (iL, iP, edge id)
	std::vector<int> cnt(Pall + 1, 0), byP(E);
	for (int u = 0; u < E; u++) cnt[IP(u) + 1]++;
	for (int p = 0; p < Pall; p++) cnt[p + 1] += cnt[p];
	for (int u = 0; u < E; u++) byP[cnt[IP(u)]++] = u;
	std::vector<int> lmPtrG(Lall + 1, 0);
	for (int u = 0; u < E; u++) lmPtrG[IL(u) + 1]++;
	for (int l = 0; l < Lall; l++) lmPtrG[l + 1] += lmPtrG[l];
	std::vector<int> orderG(E);
	{
		std::vector<int> fill(lmPtrG.begin(), lmPtrG.end() - 1);
		for (int k = 0; k < E; k++) { const int u = byP[k]; orderG[fill[IL(u)]++] = u; }
	}

	// 2. Hpl CSC (global): block index = rank of the edge among free-free edges in canonical order
	S.hplColPtr.assign(numL + 1, 0);
	S.edge2Hpl.assign(E, -1);
	std::vector<int> hplLmG;
	S.hplRowInd.reserve(E); hplLmG.reserve(E);
	for (int k = 0; k < E; k++) {
		const int u = orderG[k];
		const int ip = IP(u), il = IL(u);
		if (ip < numP && il < numL) {
			S.edge2Hpl[u] = (int)S.hplRowInd.size();
			S.hplRowInd.push_back(ip);
			hplLmG.push_back(il);
			S.hplColPtr[il + 1]++;
		}
	}
	for (int l = 0; l < numL; l++) S.hplColPtr[l + 1] += S.hplColPtr[l];
	S.nhpl = (int)S.hplRowInd.size();

	// 3. landmark shard of this rank, balanced by edge count, snapped to landmark boundaries
	auto boundary = [&](int r) {
		if (r <= 0) return 0;
		if (r >= world) return Lall;
		const long long target = (long long)E * r / world;
		return (int)(std::lower_bound(lmPtrG.begin(), lmPtrG.end(), (int)target) - lmPtrG.begin());
	};
	S.lmBeg = std::min(boundary(rank), Lall);
	S.lmEnd = std::min(std::max(boundary(rank + 1), S.lmBeg), Lall);
	const int kBeg = lmPtrG[S.lmBeg], kEnd = lmPtrG[S.lmEnd];
	S.eLocal = kEnd - kBeg;
	auto hplAt = [&](int l) { return l < numL ? S.hplColPtr[l] : S.nhpl; };
	S.hplBase = hplAt(S.lmBeg);
	S.nhplLocal = hplAt(S.lmEnd) - S.hplBase;
	S.order.resize(S.eLocal); S.e_ip.resize(S.eLocal); S.e_il.resize(S.eLocal); S.e_hpl.resize(S.eLocal);
	{
		int rankFF = 0;   // rank among the shard's free-free edges; edges without a block store -1-rank
		for (int k = kBeg; k < kEnd; k++) {
			const int u = orderG[k], e = k - kBeg;
			S.order[e] = u;
			S.e_ip[e] = IP(u) | (u >= E2 ? (int)0x80000000u : 0);
			S.e_il[e] = IL(u);
			if (S.edge2Hpl[u] >= 0) { S.e_hpl[e] = S.edge2Hpl[u] - S.hplBase; rankFF = S.e_hpl[e] + 1; }
			else S.e_hpl[e] = -1 - rankFF;
		}
	}
	S.lmPtr.resize(Lall + 1);
	for (int l = 0; l <= Lall; l++) S.lmPtr[l] = std::min(std::max(lmPtrG[l], kBeg), kEnd) - kBeg;
	S.hplLm.assign(hplLmG.begin() + S.hplBase, hplLmG.begin() + S.hplBase + S.nhplLocal);

	// 4. landmark tiles: whole landmarks, <= tileEdges edges and <= tileEdges landmarks per tile;
	//    a landmark with more edges than that gets a tile of its own
	{
		int l = S.lmBeg;
		while (l < S.lmEnd) {
			S.tileLm.push_back(l);
			int edges = 0, n = 0;
			while (l < S.lmEnd && n < tileEdges) {
				const int d = S.lmPtr[l + 1] - S.lmPtr[l];
				if (n > 0 && edges + d > tileEdges) break;
				edges += d; n++; l++;
				if (edges >= tileEdges) break;
			}
		}
		S.tileLm.push_back(S.lmEnd);
	}

	// 5. pose-major copy of the shard's edges with a free pose
	S.posePtr.assign(numP + 1, 0);
	for (int e = 0; e < S.eLocal; e++) { const int ip = S.e_ip[e] & 0x7fffffff; if (ip < numP) S.posePtr[ip + 1]++; }
	for (int p = 0; p < numP; p++) S.posePtr[p + 1] += S.posePtr[p];
	S.p_src.resize(S.posePtr[numP]); S.p_il.resize(S.posePtr[numP]);
	{
		std::vector<int> fill(S.posePtr.begin(), S.posePtr.end() - 1);
		for (int e = 0; e < S.eLocal; e++) {
			const int ip = S.e_ip[e] & 0x7fffffff;
			if (ip < numP) {
				const int pos = fill[ip]++;
				S.p_src[pos] = e;
				S.p_il[pos] = S.e_il[e] | (S.e_ip[e] & (int)0x80000000u);
			}
		}
	}

	// 6. Hsc upper pattern (global) + destination-sorted product list (shard's landmarks)
	std::vector<int> rowPtrH(numP + 1, 0), rowList(S.nhpl);
	for (int h = 0; h < S.nhpl; h++) rowPtrH[S.hplRowInd[h] + 1]++;
	for (int p = 0; p < numP; p++) rowPtrH[p + 1] += rowPtrH[p];
	{
		std::vector<int> fill(rowPtrH.begin(), rowPtrH.end() - 1);
		for (int h = 0; h < S.nhpl; h++) rowList[fill[S.hplRowInd[h]]++] = h;
	}
	std::vector<int> mark(numP, 0), cntLoc(numP, 0), touched;
	std::vector<int> prodCount;
	S.hscRowPtr.assign(numP + 1, 0);
	S.nmul = 0; S.nmulLocal = 0;
	for (int a = 0; a < numP; a++) {
		touched.clear();
		touched.push_back(a); mark[a] = 1;     // the diagonal block always exists
		for (int x = rowPtrH[a]; x < rowPtrH[a + 1]; x++) {
			const int i = rowList[x];
			const int l = hplLmG[i];
			const bool local = l >= S.lmBeg && l < S.lmEnd;
			const int cend = S.hplColPtr[l + 1];
			for (int j = i; j < cend; j++) {
				const int b = S.hplRowInd[j];
				if (!mark[b]) { mark[b] = 1; touched.push_back(b); }
				if (local) cntLoc[b]++;
			}
			S.nmul += cend - i;
		}
		std::sort(touched.begin(), touched.end());
		for (int b : touched) {
			S.blkRow.push_back(a); S.blkCol.push_back(b);
			prodCount.push_back(cntLoc[b]);
			S.nmulLocal += cntLoc[b];
			mark[b] = 0; cntLoc[b] = 0;
		}
		S.hscRowPtr[a + 1] = (int)S.blkRow.size();
	}
	S.nblk = (int)S.blkRow.size();
	S.hscColInd = S.blkCol;
	if (S.nmulLocal > 0x7fffffffLL) { *err = "build_structure: more than 2^31 block products in one shard"; return false; }
	S.prodPtr.assign(S.nblk + 1, 0);
	for (int k = 0; k < S.nblk; k++) S.prodPtr[k + 1] = S.prodPtr[k] + prodCount[k];
	S.prodI.resize((size_t)S.nmulLocal); S.prodJ.resize((size_t)S.nmulLocal);
	{
		std::vector<int> off(numP, 0);
		for (int a = 0; a < numP; a++) {
			for (int k = S.hscRowPtr[a]; k < S.hscRowPtr[a + 1]; k++) off[S.blkCol[k]] = S.prodPtr[k];
			for (int x = rowPtrH[a]; x < rowPtrH[a + 1]; x++) {
				const int i = rowList[x];
				const int l = hplLmG[i];
				if (l < S.lmBeg || l >= S.lmEnd) continue;
				const int cend = S.hplColPtr[l + 1];
				for (int j = i; j < cend; j++) {
					const int pos = off[S.hplRowInd[j]]++;
					S.prodI[pos] = i - S.hplBase;
					S.prodJ[pos] = j - S.hplBase;
				}
			}
		}
	}

	// 7. symmetric-full BSR: row r = [ (a,r) transposed entries, a<r ascending ] ++ [ (r,b) upper entries ]
	{
		std::vector<int> cntT(numP, 0);
		for (int k = 0; k < S.nblk; k++) if (S.blkRow[k] != S.blkCol[k]) cntT[S.blkCol[k]]++;
		S.fRowPtr.assign(numP + 1, 0);
		for (int r = 0; r < numP; r++) S.fRowPtr[r + 1] = S.fRowPtr[r] + cntT[r] + (S.hscRowPtr[r + 1] - S.hscRowPtr[r]);
		S.nfull = S.fRowPtr[numP];
		S.fColInd.resize(S.nfull); S.u2f.resize(S.nblk); S.u2fT.resize(S.nblk);
		std::vector<int> fillT(numP, 0);
		for (int k = 0; k < S.nblk; k++) {
			const int a = S.blkRow[k], b = S.blkCol[k];
			const int pos = S.fRowPtr[a] + cntT[a] + (k - S.hscRowPtr[a]);
			S.fColInd[pos] = b; S.u2f[k] = pos;
			if (a != b) {
				const int posT = S.fRowPtr[b] + fillT[b]++;
				S.fColInd[posT] = a; S.u2fT[k] = posT;
			} else S.u2fT[k] = pos;
		}
	}
	return true;
}

// ---- host side of the PCG setup ---------------------------------------------------------------------------------
void build_pcg_partition(int numP, int nfull, const std::vector<int>& fRowPtr, const std::vector<int>& fColInd, int G, PcgPartition& P,
	int maxRows)
{
	P = PcgPartition();
	P.G = G;
	// contiguous row ranges balanced by block count
	std::vector<int>& rows = P.rows;
	rows.assign(G + 1, 0);
	{
		int r = 0;
		for (int c = 0; c < G; c++) {
			rows[c] = r;
			const long long target = (long long)nfull * (c + 1) / G;
			const int minRows = 1, remainingCtas = G - c - 1;
			int end = r + minRows;
			if (maxRows > 0) end = std::max(end, numP - remainingCtas * maxRows);   // the CTAs after this one can take the rest
			while (end < numP - remainingCtas && fRowPtr[end] < target && (maxRows <= 0 || end - r < maxRows)) end++;
			r = std::min(end, numP - remainingCtas);
		}
		rows[G] = numP;
	}
	P.nptr.assign(G + 1, 0);
	P.local.resize(nfull);
	P.ncol.reserve((size_t)nfull / 4 + numP);
	// per CTA: the distinct columns of its blocks (mark), sorted; pos[j] = place of column j in that list -> the local index of
	// every block is one lookup (this runs on the host inside set_problem: 81 k blocks of ba_kitti_00 in 0.2 ms)
	std::vector<int> mark(numP, -1), pos(numP, 0), cols;
	cols.reserve(1024);
	for (int c = 0; c < G; c++) {
		const int n0 = fRowPtr[rows[c]], n1 = fRowPtr[rows[c + 1]];
		cols.clear();
		for (int n = n0; n < n1; n++) {
			const int j = fColInd[n];
			if (mark[j] != c) { mark[j] = c; cols.push_back(j); }
		}
		std::sort(cols.begin(), cols.end());
		P.nptr[c] = (int)P.ncol.size();
		for (size_t k = 0; k < cols.size(); k++) { pos[cols[k]] = (int)k; P.ncol.push_back(cols[k]); }
		// the diagonal block of each own row is encoded as -1-loc (A^_ii = I is applied implicitly)
		for (int r = rows[c]; r < rows[c + 1]; r++)
			for (int n = fRowPtr[r]; n < fRowPtr[r + 1]; n++) {
				const int j = fColInd[n], loc = pos[j];
				P.local[n] = j == r ? -1 - loc : loc;
			}
		P.maxRows = std::max(P.maxRows, rows[c + 1] - rows[c]);
		P.needMax = std::max(P.needMax, (int)cols.size());
		P.blkMax = std::max(P.blkMax, n1 - n0);
	}
	P.nptr[G] = (int)P.ncol.size();
}

void build_coarse_partition(int numP, const PcgPartition& P, int maxAgg, CoarsePartition& C, int apc)
{
	C = CoarsePartition();
	const int G = P.G;
	if (apc > 1) {
		// apc aggregates per CTA: the CTA's rows in apc contiguous groups balanced by row count (a CTA with fewer rows: no partition)
		for (int c = 0; c < G; c++) if (P.rows[c + 1] - P.rows[c] < apc) return;
		C.gs = 1; C.apc = apc; C.A = G * apc;
		C.aggRow.assign(C.A + 1, numP);
		for (int c = 0; c < G; c++)
			for (int j = 0; j < apc; j++) C.aggRow[c * apc + j] = P.rows[c] + (P.rows[c + 1] - P.rows[c]) * j / apc;
	} else {
		const int gs = (G + maxAgg - 1) / maxAgg;
		C.gs = gs; C.A = (G + gs - 1) / gs;
		C.aggRow.assign(C.A + 1, numP);
		for (int ag = 0; ag < C.A; ag++) C.aggRow[ag] = P.rows[std::min(ag * gs, G)];
	}
	const int A = C.A;
	C.rowAgg.assign(numP, 0);
	for (int ag = 0; ag < A; ag++) for (int r = C.aggRow[ag]; r < C.aggRow[ag + 1]; r++) C.rowAgg[r] = ag;
	C.naPtr.assign(G + 1, 0);
	C.needAgg.resize(P.ncol.size());
	int maxNA = 0;
	// per CTA: the distinct aggregates of its needed columns (mark), ascending; pos[a] = place of aggregate a in that list
	std::vector<int> mark(A, -1), pos(A, 0), ags;
	for (int c = 0; c < G; c++) {
		ags.clear();
		for (int k = P.nptr[c]; k < P.nptr[c + 1]; k++) {
			const int a = C.rowAgg[P.ncol[k]];
			if (mark[a] != c) { mark[a] = c; ags.push_back(a); }
		}
		std::sort(ags.begin(), ags.end());
		C.naPtr[c] = (int)C.naList.size();
		for (size_t k = 0; k < ags.size(); k++) pos[ags[k]] = (int)k;
		for (int k = P.nptr[c]; k < P.nptr[c + 1]; k++) C.needAgg[k] = pos[C.rowAgg[P.ncol[k]]];
		C.naList.insert(C.naList.end(), ags.begin(), ags.end());
		maxNA = std::max(maxNA, (int)ags.size());
	}
	C.naPtr[G] = (int)C.naList.size();
	C.maxNeedAgg = std::max(maxNA, 1);
}

void build_coarse_lists(int numP, int nfull, const std::vector<int>& fRowPtr, const std::vector<int>& fColInd, CoarsePartition& C)
{
	// fine blocks of every coarse block (lower triangle), ascending -> fixed-order sums in k_coarse_assemble
	const int A = C.A, nblkP = A * (A + 1) / 2;
	C.rowOf.resize(nfull);
	C.cbPtr.assign(nblkP + 1, 0);
	std::vector<int> cbOf(nfull);                     // coarse block of every fine block, -1 above the coarse diagonal
	for (int i = 0; i < numP; i++) {
		const int ai = C.rowAgg[i], base = ai * (ai + 1) / 2;
		for (int n = fRowPtr[i]; n < fRowPtr[i + 1]; n++) {
			C.rowOf[n] = i;
			const int aj = C.rowAgg[fColInd[n]];
			const int cb = ai >= aj ? base + aj : -1;
			cbOf[n] = cb;
			if (cb >= 0) C.cbPtr[cb + 1]++;
		}
	}
	for (int cb = 0; cb < nblkP; cb++) C.cbPtr[cb + 1] += C.cbPtr[cb];
	C.cbList.resize(C.cbPtr[nblkP]);
	std::vector<int> fill(C.cbPtr.begin(), C.cbPtr.end() - 1);
	for (int n = 0; n < nfull; n++) { const int cb = cbOf[n]; if (cb >= 0) C.cbList[fill[cb]++] = n; }
}

const char* check_pcg_partition(int numP, int nfull, const std::vector<int>& fRowPtr, const std::vector<int>& fColInd,
	const PcgPartition& P, const CoarsePartition& C)
{
	const int G = P.G;
	if (G < 1 || (int)P.rows.size() != G + 1 || P.rows[0] != 0 || P.rows[G] != numP) return "rows do not cover [0, numP)";
	for (int c = 0; c < G; c++) if (P.rows[c + 1] <= P.rows[c]) return "a CTA without rows";
	for (int c = 0; c < G; c++) {
		const int* nc = P.ncol.data() + P.nptr[c];
		const int nn = P.nptr[c + 1] - P.nptr[c];
		for (int k = 1; k < nn; k++) if (nc[k] <= nc[k - 1]) return "need list not strictly ascending";
		for (int r = P.rows[c]; r < P.rows[c + 1]; r++) {
			if (!std::binary_search(nc, nc + nn, r)) return "own row missing from the need list";
			bool diag = false;
			for (int n = fRowPtr[r]; n < fRowPtr[r + 1]; n++) {
				const int loc = P.local[n], j = fColInd[n];
				const int pos = loc < 0 ? -1 - loc : loc;
				if (pos < 0 || pos >= nn || nc[pos] != j) return "local index does not point at the block's column";
				if ((loc < 0) != (j == r)) return "diagonal encoding wrong";
				diag |= j == r;
			}
			if (!diag) return "row without a diagonal block";
		}
		if (nn > P.needMax || P.rows[c + 1] - P.rows[c] > P.maxRows || fRowPtr[P.rows[c + 1]] - fRowPtr[P.rows[c]] > P.blkMax) return "maxima too small";
	}
	// coarse level
	const int A = C.A, apc = C.apc;
	if (A < 1 || (int)C.aggRow.size() != A + 1 || C.aggRow[0] != 0 || C.aggRow[A] != numP) return "aggregates do not cover [0, numP)";
	if (apc < 1 || (apc > 1 && (C.gs != 1 || A != G * apc))) return "aggregates per CTA inconsistent";
	for (int a = 0; a < A; a++) {
		if (C.aggRow[a + 1] <= C.aggRow[a]) return "empty aggregate";
		if (apc == 1 && C.aggRow[a] != P.rows[std::min(a * C.gs, G)]) return "aggregate not aligned with a CTA boundary";
		if (apc > 1) {
			// aggregate a is part j of CTA c: it starts at the CTA's first row when j == 0 and never leaves the CTA
			const int c = a / apc, j = a - c * apc, n = P.rows[c + 1] - P.rows[c];
			if ((j == 0 && C.aggRow[a] != P.rows[c]) || C.aggRow[a + 1] > P.rows[c + 1]) return "aggregate straddles two CTAs";
			if (std::abs((C.aggRow[a + 1] - C.aggRow[a]) - n / apc) > 1) return "aggregates of a CTA not balanced by row count";
		}
		for (int r = C.aggRow[a]; r < C.aggRow[a + 1]; r++) if (C.rowAgg[r] != a) return "rowAgg inconsistent";
	}
	for (int c = 0; c < G; c++) {
		const int* al = C.naList.data() + C.naPtr[c];
		const int na = C.naPtr[c + 1] - C.naPtr[c];
		if (na < 1 || na > C.maxNeedAgg) return "aggregate list size";
		for (int k = 1; k < na; k++) if (al[k] <= al[k - 1]) return "aggregate list not ascending";
		for (int k = P.nptr[c]; k < P.nptr[c + 1]; k++) {
			const int pos = C.needAgg[k];
			if (pos < 0 || pos >= na || al[pos] != C.rowAgg[P.ncol[k]]) return "needAgg does not point at the column's aggregate";
		}
		if (C.rowAgg[P.rows[c]] != c / C.gs * apc) return "a CTA's first row is not in aggregate cta / gs * apc";
	}
	if (!C.cbPtr.empty()) {
		const int nblkP = A * (A + 1) / 2;
		if ((int)C.cbPtr.size() != nblkP + 1) return "cbPtr size";
		long long lower = 0;
		for (int n = 0; n < nfull; n++) if (C.rowAgg[C.rowOf[n]] >= C.rowAgg[fColInd[n]]) lower++;
		if ((long long)C.cbList.size() != lower || C.cbPtr[nblkP] != (int)lower) return "coarse lists do not hold every lower block exactly once";
		for (int ib = 0; ib < A; ib++)
			for (int jb = 0; jb <= ib; jb++) {
				const int cb = ib * (ib + 1) / 2 + jb;
				for (int k = C.cbPtr[cb]; k < C.cbPtr[cb + 1]; k++) {
					const int n = C.cbList[k];
					if (n < 0 || n >= nfull || C.rowAgg[C.rowOf[n]] != ib || C.rowAgg[fColInd[n]] != jb) return "block in the wrong coarse list";
					if (k > C.cbPtr[cb] && C.cbList[k - 1] >= n) return "coarse list not ascending";
				}
			}
	}
	return nullptr;
}

void build_pcg5_plan(int numP, int nfull, const std::vector<int>& fRowPtr, const std::vector<int>& fColInd, int world, int numSMs, int maxAgg,
	int maxRowsPerCta, Pcg5Plan& plan, const PcgPartition* same, int apc)
{
	plan = Pcg5Plan();
	plan.world = world;
	if (numP < 1 || world < 1 || world > 8 || apc < 1 || (apc > 1 && world > 1)) return;
	// CTAs per GPU: about eight rows each
	int G = std::max(1, std::min(numSMs, (numP / world + 7) / 8));
	if (world * G > numP) G = std::max(1, numP / world);
	// one aggregate per group of gs CTAs (at most maxAgg of them), or apc aggregates per CTA (maxAgg does not apply)
	const int gs = apc > 1 ? 1 : (world * G + maxAgg - 1) / maxAgg;
	G = std::max(gs, G / gs * gs);
	const int Gt = world * G, A = Gt / gs * apc;
	if (Gt > numP || A < 1 || G > numSMs) return;
	if (same && same->G == Gt && (int)same->rows.size() == Gt + 1 && same->rows[Gt] == numP && (int)same->local.size() == nfull) plan.P = *same;
	else build_pcg_partition(numP, nfull, fRowPtr, fColInd, Gt, plan.P);
	// balanced by blocks, a CTA may get more rows than the row sums can take (a large graph on a GPU with fewer SMs, e.g. 10 000 poses
	// on an H100's 132): balance again with the row count capped
	if (plan.P.maxRows > maxRowsPerCta) build_pcg_partition(numP, nfull, fRowPtr, fColInd, Gt, plan.P, maxRowsPerCta);
	build_coarse_partition(numP, plan.P, A, plan.C, apc);
	if (plan.C.gs != gs || plan.C.A != A || plan.P.maxRows > maxRowsPerCta) return;
	build_coarse_lists(numP, nfull, fRowPtr, fColInd, plan.C);
	plan.rowPeers.assign(numP, 0);
	if (world > 1) {
		std::vector<int> rowRank(numP, 0);
		for (int c = 0; c < Gt; c++) for (int r = plan.P.rows[c]; r < plan.P.rows[c + 1]; r++) rowRank[r] = c / G;
		for (int c = 0; c < Gt; c++)
			for (int k = plan.P.nptr[c]; k < plan.P.nptr[c + 1]; k++) {
				const int j = plan.P.ncol[k];
				if (rowRank[j] != c / G) plan.rowPeers[j] |= (unsigned char)(1u << (c / G));
			}
	}
	plan.G = G; plan.gs = gs; plan.A = A; plan.apc = apc;
	plan.ok = true;
}

const char* check_pcg5_plan(int numP, int nfull, const std::vector<int>& fRowPtr, const std::vector<int>& fColInd, const Pcg5Plan& plan)
{
	if (!plan.ok) return "plan not ok";
	const int G = plan.G, W = plan.world, Gt = G * W, gs = plan.gs, apc = plan.apc;
	if (plan.P.G != Gt) return "virtual CTA count";
	if (apc != plan.C.apc || (apc > 1 && (gs != 1 || W != 1))) return "aggregates per CTA";
	if (G % gs != 0 || plan.A * gs != Gt * apc) return "aggregates do not tile the ranks";
	const char* bad = check_pcg_partition(numP, nfull, fRowPtr, fColInd, plan.P, plan.C);
	if (bad) return bad;
	// every aggregate lies inside one rank
	for (int a = 0; a < plan.A; a++) {
		const int c0 = a / apc * gs, c1 = c0 + gs - 1;
		if (c0 / G != c1 / G) return "aggregate straddles two ranks";
	}
	// rowPeers: exactly the ranks (not the owner) with a CTA that needs the row
	std::vector<int> rowRank(numP, 0);
	for (int c = 0; c < Gt; c++) for (int r = plan.P.rows[c]; r < plan.P.rows[c + 1]; r++) rowRank[r] = c / G;
	std::vector<unsigned> want(numP, 0);
	for (int i = 0; i < numP; i++)
		for (int n = fRowPtr[i]; n < fRowPtr[i + 1]; n++) { const int j = fColInd[n]; if (rowRank[j] != rowRank[i]) want[j] |= 1u << rowRank[i]; }
	for (int j = 0; j < numP; j++) {
		if ((unsigned)plan.rowPeers[j] != want[j]) return "rowPeers differs from the ranks whose rows couple to the row";
		if (plan.rowPeers[j] & (1u << rowRank[j])) return "rowPeers names the owner";
	}
	return nullptr;
}

}  // namespace cuba_b200
