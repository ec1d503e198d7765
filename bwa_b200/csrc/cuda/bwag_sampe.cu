/* bwag_sampe.cu -- `bwa-b200 sampe`: the device half of the reference's bwa_sai2sam_pe_core (bwape.c:260-711).
 *
 *   P1/P2  k_pe_pos     after K2 (k_sa) resolved the rows in place, one lane per row: bwa_sa2pos with the two reference lengths
 *                       the host asks for (len + the chosen hit's ref_shift for the pairing candidates, len + the interval's
 *                       ref_shift for XA; the main hits of P1 ask for one)
 *   P5     k_pe_global  one warp per accepted local alignment of the mate rescue (bwa_sw_core, bwape.c:434): ksw_global with
 *                       band 50 over [qb, qe] x [tb, te] and the raw CIGAR, none of bwa_refine_gapped_core's fix-ups; the local
 *                       alignments themselves are K6 (k_localsw*, bwag_localsw.cu)
 *   P6     k_se_refine  (bwag_samse.cu) unchanged: the gapped refinement of the hits the pairing left in place and of XA
 *   P7     k_pe_text    one lane per read, twice around a scan, as samse's S4: bwa_print_sam1 with a mate (bwase.c:386-499)
 * Pairs are reads 2i (end 1) and 2i + 1 (end 2) of the batch. */
#include "bwag_dev.cuh"
#include "bwag_kernels.h"
#include "bwag_ksw.cuh"
#include "bwag_se.cuh"

__global__ void k_pe_pos(PePosArgs a)
{
	for (i64 i = (i64)blockIdx.x * blockDim.x + threadIdx.x; i < a.n; i += (i64)gridDim.x * blockDim.x) {
		const i64 pos_f = a.rows[i];
		for (int k = 0; k < 2; ++k) {
			uint8_t st;
			a.pos[2 * i + k] = se_sa2pos(a.l_pac, pos_f, a.ref_len[2 * i + k], &st);
			a.strand[2 * i + k] = st;
		}
	}
}

/* one warp per task: score (eh[qlen].h of ksw_global2) and the CIGAR (len << 4 | op) at cig_off */
__global__ void __launch_bounds__(SE_THREADS) k_pe_global(DevIndex ix, PeGlbArgs a)
{
	const int lane = threadIdx.x & 31;
	const i64 wid = ((i64)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
	int *H = a.eh + wid * (i64)(2 * (a.cap_q + 2)), *E = H + a.cap_q + 2;
	uint8_t *rs = a.rseq + wid * (i64)a.cap_r, *z = a.z + wid * a.cap_z;
	__shared__ int8_t s_mat[32];
	if (threadIdx.x < 32) s_mat[threadIdx.x] = threadIdx.x >= 25 ? -1 : threadIdx.x % 5 == 4 || threadIdx.x >= 20 ? -1 : threadIdx.x / 5 == threadIdx.x % 5 ? 1 : -3;   /* bwa_fill_scmat(1, 3) */
	__syncthreads();
	u64 cells = 0;
	for (;;) {
		int t = 0;
		if (lane == 0) t = atomicAdd(a.next_task, 1);
		t = __shfl_sync(FULL_MASK, t, 0);
		if (t >= a.n_tasks) break;
		const bwag_pe_gtask_t tk = a.tasks[t];
		const int qlen = tk.qlen, tlen = tk.tlen;
		for (int x = lane; x < tlen; x += 32) rs[x] = (uint8_t)bwag_pac_base(ix.pac, tk.t_beg + x);
		__syncwarp();
		const int n_col = qlen < 2 * 50 + 1 ? qlen : 2 * 50 + 1;
		const int score = warp_ksw_global(lane, qlen, a.pool + tk.q_beg, tlen, rs, s_mat, 5, 1, 5, 1, 50, H, E, z, n_col, &cells);
		if (lane == 0) {
			bwag_pe_gres_t r;
			r.score = score; r.cig_off = a.res[t].cig_off;
			r.n_cigar = ksw_backtrack(z, n_col, tlen, qlen, 50, a.cig + r.cig_off);
			a.res[t] = r;
		}
		__syncwarp();
	}
	if (lane == 0 && cells) atomicAdd(a.cells, cells);
}

/* one end after refinement and bwa_correct_trimmed: its position, strand and corrected CIGAR */
struct PeEnd {
	bool mapped; int type, strand, full_len; i64 pos; const u32 *cig; int n_cigar; SeCig ec;
	__device__ __forceinline__ i64 end() const   /* pos_end */
	{
		if (!ec.n) return pos + full_len;
		i64 x = pos;
		for (int k = 0; k < ec.n; ++k) { const u32 cv = ec.at(k); if (se_op(cv) == 0 || se_op(cv) == 2) x += se_len(cv); }
		return x;
	}
	__device__ __forceinline__ i64 pos5() const { return strand ? end() : pos; }
};

__device__ __forceinline__ PeEnd pe_end(const SeArgs &a, const bwag_pe_read_t *pe, int r)
{
	const bwag_se_read_t p = a.reads[r];
	PeEnd e;
	e.type = p.type; e.mapped = p.type != 0; e.strand = a.strand[r]; e.pos = a.pos[r];
	e.full_len = (int)(a.off[r + 1] - a.off[r]);
	e.cig = 0; e.n_cigar = 0;
	if (p.type == 3) { e.cig = a.cig + pe[r].cig_off; e.n_cigar = pe[r].n_cig; }
	else if (e.mapped) {
		const int t = a.main_task[r];
		if (t >= 0) { e.cig = a.cig + a.tasks[t].cig_off; e.n_cigar = a.ncig[t]; e.pos += a.tshift[t]; }
	}
	e.ec = se_corrected(e.cig, e.n_cigar, p.len, e.full_len, e.strand);   /* every read, the unmapped ones on the forward strand */
	return e;
}

__global__ void k_pe_text(DevIndex ix, SeArgs a, const bwag_pe_read_t *pe, int write)
{
	for (int r = blockIdx.x * blockDim.x + threadIdx.x; r < a.n_reads; r += gridDim.x * blockDim.x) {
		const bwag_se_read_t p = a.reads[r];
		const i64 o0 = write ? a.tbeg[r] : 0;
		SeOut o = { write ? a.text + o0 : 0, 0 };
		const uint8_t *read = a.codes + a.off[r];
		const PeEnd P = pe_end(a, pe, r), M = pe_end(a, pe, r ^ 1);
		const int full_len = P.full_len, len = p.len;
		int flag = pe[r].flag, strand = P.strand;
		i64 len_a;
		if (P.mapped || M.mapped) {
			i64 pos;
			int j, seqid;
			if (!P.mapped) { pos = M.pos; strand = M.strand; flag |= 4; j = 1; }
			else { pos = P.pos; j = (int)(P.end() - pos); }
			const int nn = se_cnt_ambi(a, pos, j, &seqid);
			if (P.mapped && pos + j - a.ctg.off[seqid] > a.ctg.len[seqid]) flag |= 4;   /* bridges two adjacent contigs */
			if (strand) flag |= 16;
			if (M.mapped) { if (M.strand) flag |= 32; } else flag |= 8;
			o.c('\t'); o.d(flag); o.c('\t');
			o.s(a.ctg.names + a.ctg.name_off[seqid], a.ctg.name_off[seqid + 1] - a.ctg.name_off[seqid]);
			o.c('\t'); o.d((int)(pos - a.ctg.off[seqid] + 1)); o.c('\t'); o.d(p.mapq); o.c('\t');
			if (P.ec.n) for (int k = 0; k < P.ec.n; ++k) { const u32 cv = P.ec.at(k); o.d(se_len(cv)); o.c("MIDS"[se_op(cv)]); }
			else if (!P.mapped) o.c('*');
			else { o.d(full_len); o.c('M'); }
			if (M.mapped) {
				int mid;
				se_cnt_ambi(a, M.pos, M.full_len, &mid);
				o.c('\t');
				if (mid == seqid) o.c('=');
				else o.s(a.ctg.names + a.ctg.name_off[mid], a.ctg.name_off[mid + 1] - a.ctg.name_off[mid]);
				o.c('\t'); o.d((int)(M.pos - a.ctg.off[mid] + 1)); o.c('\t');
				o.d(P.mapped && mid == seqid ? M.pos5() - P.pos5() : 0); o.c('\t');
			} else { o.s("\t=\t"); o.d((int)(pos - a.ctg.off[seqid] + 1)); o.s("\t0\t"); }
			if (!strand) for (int i = 0; i < full_len; ++i) o.c("ACGTN\0"[read[i]]);
			else for (int i = full_len - 1; i >= 0; --i) o.c("TGCAN\0"[read[i]]);
			o.c('\t');
			len_a = o.n;
			if (a.l_rg) { o.s("\tRG:Z:"); o.s(a.rg, a.l_rg); }
			if (p.l_bc) { o.s("\tBC:Z:"); o.s(a.bc + p.bc_off, p.l_bc); }
			if (p.clip_len < full_len) { o.s("\tXC:i:"); o.d(p.clip_len); }
			if (P.mapped) {
				const SeRead q = { read, len, P.strand != 0, pe[r].comp != 0 };   /* the read's own .sai decides its rseq; NM vs CM is .sai 2's */
				SeOut md_count = { 0, 0 };
				const int nm = write ? a.nm[r] : se_md(ix, a.ctg.l_pac, P.cig, P.n_cigar, q, P.pos, &md_count);
				if (!write) a.nm[r] = nm;
				char xt = "NURM"[p.type & 3];
				if (nn > 10) xt = 'N';
				o.s("\tXT:A:"); o.c(xt);
				o.s((a.mode & BWAG_SE_COMPREAD) ? "\tNM:i:" : "\tCM:i:"); o.d(nm & 0xfff);
				if (nn) { o.s("\tXN:i:"); o.d(nn); }
				o.s("\tSM:i:"); o.d(pe[r].seq_q);
				o.s("\tAM:i:"); o.d(M.mapped ? (pe[r ^ 1].seq_q < pe[r].seq_q ? pe[r ^ 1].seq_q : pe[r].seq_q) : 0);
				if (p.type != 3) {   /* X0 and X1 are not available for a mate-rescued alignment */
					o.s("\tX0:i:"); o.d((int)p.c1);
					if ((int)p.c1 <= a.max_top2) { o.s("\tX1:i:"); o.d((int)p.c2); }
				}
				o.s("\tXM:i:"); o.d(p.n_mm); o.s("\tXO:i:"); o.d(p.n_gapo); o.s("\tXG:i:"); o.d(p.n_gapo + p.n_gape);
				o.s("\tMD:Z:");
				if (write) se_md(ix, a.ctg.l_pac, P.cig, P.n_cigar, q, P.pos, &o);
				else o.n += md_count.n;
				/* XA: the candidates the host kept, refined if gapped */
				for (int k = 0; k < p.n_multi; ++k) {
					const i64 s = p.multi_beg + k;
					if (k == 0) o.s("\tXA:Z:");
					const int mt = a.multi_task[s];
					const u32 *mc = mt >= 0 ? a.cig + a.tasks[mt].cig_off : 0;
					const int mn = mt >= 0 ? a.ncig[mt] & 0x7fff : 0;   /* bwt_multi1_t keeps n_cigar in 15 bits */
					const i64 mp = a.mpos[s] + (mt >= 0 ? a.tshift[mt] : 0);
					i64 e = mp;
					if (mc) { for (int x = 0; x < mn; ++x) { const int op = se_op(mc[x]); if (op == 0 || op == 2) e += se_len(mc[x]); } }
					else e += full_len;
					int sid;
					se_cnt_ambi(a, mp, (int)(e - mp), &sid);
					o.s(a.ctg.names + a.ctg.name_off[sid], a.ctg.name_off[sid + 1] - a.ctg.name_off[sid]);
					o.c(','); o.c(a.mstrand[s] ? '-' : '+'); o.d((int)(mp - a.ctg.off[sid] + 1)); o.c(',');
					if (mc) for (int x = 0; x < mn; ++x) { o.d(se_len(mc[x])); o.c("MIDS"[se_op(mc[x])]); }
					else { o.d(full_len); o.c('M'); }
					o.c(','); o.d((int)a.multi[s].gap + (int)a.multi[s].mm); o.c(';');
				}
			}
		} else {
			flag |= 4 | 8;
			o.c('\t'); o.d(flag); o.s("\t*\t0\t0\t*\t*\t0\t0\t");
			for (int i = 0; i < full_len; ++i) o.c("ACGTN\0"[read[i]]);
			o.c('\t');
			len_a = o.n;
			if (a.l_rg) { o.s("\tRG:Z:"); o.s(a.rg, a.l_rg); }
			if (p.l_bc) { o.s("\tBC:Z:"); o.s(a.bc + p.bc_off, p.l_bc); }
			if (p.clip_len < full_len) { o.s("\tXC:i:"); o.d(p.clip_len); }
		}
		if (!write) a.tlen[r] = o.n;
		else {
			bwag_samrec_t rc;
			rc.off = o0; rc.len_a = (int32_t)len_a; rc.len_b = (int32_t)(o.n - len_a);
			rc.flags = BWAG_REC_TEXT | (strand ? BWAG_REC_QREV : 0u); rc.pad = 0;
			a.rec[r] = rc;
		}
	}
}
