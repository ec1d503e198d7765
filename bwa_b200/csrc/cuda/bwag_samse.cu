/* bwag_samse.cu -- `bwa-b200 samse`: the device half of the reference's bwa_sai2sam_se_core (bwase.c:507-577) once the host has
 * chosen each read's hit (bwa_aln2seq_core, whose random draws are serial) and its mapping quality.
 *
 *   S1  k_se_rows    one lane per hit: the chosen hits' and the XA candidates' suffix-array rows, which K2 (k_sa) resolves in place;
 *   S2  k_se_pos     one lane per read: bwa_sa2pos of the chosen hit and of each candidate, and which candidates stay in XA
 *                    (bwase.c:152-162: not -1, not the chosen hit's position before its refinement);
 *   S3  k_se_refine  one warp per gapped hit: ksw_global of the searched bases against the forward reference window
 *                    [pos, pos + len + ref_shift), band max(50, 1.5 |rlen - len|), scores bwa_fill_scmat(1, 3) and gaps 5/1, with the
 *                    end fix-ups of bwa_refine_gapped_core (bwase.c:169-199): the sweep and the backtrack of K5 (bwag_ksw.cuh);
 *   S4  k_se_text    one lane per read, twice: first the exact byte lengths of the record's two parts, then, after a scan, the
 *                    record itself: bwa_print_sam1 with no mate (bwase.c:386-499), MD/NM (bwa_cal_md1) and the trimming correction
 *                    (bwa_correct_trimmed) computed on the way, by the same code in both passes.
 * The host splices the read name and QUAL into each record (bwag_samrec_t), as stage 4's writer does. */
#include "bwag_dev.cuh"
#include "bwag_kernels.h"
#include "bwag_ksw.cuh"
#include "bwag_se.cuh"

#define SE_BAND 50   /* SW_BW, bwase.c:167 */

__global__ void k_se_rows(SeArgs a)
{
	const i64 n = (i64)a.n_reads + a.n_multi;
	for (i64 i = (i64)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (i64)gridDim.x * blockDim.x)
		a.rows[i] = (i64)(i < a.n_reads ? a.reads[i].sa : a.multi[i - a.n_reads].sa);
}

__global__ void k_se_pos(SeArgs a)
{
	for (int r = blockIdx.x * blockDim.x + threadIdx.x; r < a.n_reads; r += gridDim.x * blockDim.x) {
		const bwag_se_read_t p = a.reads[r];
		i64 pos = 0;   /* bwa_cal_pac_pos_core leaves an unmatched read's position alone (0) */
		uint8_t strand = 0, mapped = p.type != 0;
		if (mapped) {
			pos = se_sa2pos(a.ctg.l_pac, a.rows[r], p.len + p.ref_shift, &strand);
			if (pos == -1) mapped = 0;
		}
		a.pos[r] = pos; a.strand[r] = strand; a.mapped[r] = mapped;
		for (int k = 0; k < p.n_multi; ++k) {
			const i64 s = p.multi_beg + k;
			uint8_t st;
			const i64 q = se_sa2pos(a.ctg.l_pac, a.rows[a.n_reads + s], p.len + a.multi[s].ref_shift, &st);
			a.mpos[s] = q; a.mstrand[s] = st; a.mkeep[s] = q != pos && q != -1;
		}
	}
}


/* S3: one warp per task; tasks whose hit turned out unmapped or left XA are skipped */
__global__ void __launch_bounds__(SE_THREADS) k_se_refine(DevIndex ix, SeArgs a)
{
	const int lane = threadIdx.x & 31;
	const i64 wid = ((i64)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
	int *H = a.eh + wid * (i64)(2 * (a.cap_q + 2)), *E = H + a.cap_q + 2;
	uint8_t *rs = a.rseq + wid * (i64)a.cap_r, *qs = a.qseq + wid * (i64)a.cap_q, *z = a.z + wid * a.cap_z;
	__shared__ int8_t s_mat[32];
	if (threadIdx.x < 32) s_mat[threadIdx.x] = threadIdx.x >= 25 ? -1 : threadIdx.x % 5 == 4 || threadIdx.x >= 20 ? -1 : threadIdx.x / 5 == threadIdx.x % 5 ? 1 : -3;   /* bwa_fill_scmat(1, 3) */
	__syncthreads();
	u64 cells = 0, n_run = 0;
	for (;;) {
		int t = 0;
		if (lane == 0) t = atomicAdd(a.next_task, 1);
		t = __shfl_sync(FULL_MASK, t, 0);
		if (t >= a.n_tasks) break;
		const SeTask tk = a.tasks[t];
		const bwag_se_read_t p = a.reads[tk.read];
		i64 pos; int strand, ref_shift;
		if (tk.slot < 0) { if (!a.mapped[tk.read]) continue; pos = a.pos[tk.read]; strand = a.strand[tk.read]; ref_shift = p.ref_shift; }
		else { if (!a.mkeep[tk.slot]) continue; pos = a.mpos[tk.slot]; strand = a.mstrand[tk.slot]; ref_shift = a.multi[tk.slot].ref_shift; }
		const int len = p.len;
		const i64 re = pos + len + ref_shift;
		if (re > ix.l_pac) {   /* assert(re <= l_pac) of the reference */
			if (lane == 0) atomicMax(a.past_end, a.n_reads - tk.read);
			continue;
		}
		const int rlen = (int)(re - pos);
		const uint8_t *read = a.codes + a.off[tk.read];
		const bool comp = (a.mode & BWAG_SE_COMPREAD) != 0;
		for (int x = lane; x < rlen; x += 32) rs[x] = (uint8_t)bwag_pac_base(ix.pac, pos + x);
		for (int x = lane; x < len; x += 32) {   /* the read, or rseq: reversed, complemented under COMPREAD (seq_reverse) */
			uint8_t c = strand ? read[len - 1 - x] : read[x];
			if (strand && comp && c < 4) c = 3 - c;
			qs[x] = c;
		}
		__syncwarp();
		int w = (int)(abs(rlen - len) * 1.5);
		w = SE_BAND > w ? SE_BAND : w;
		const int n_col = len < 2 * w + 1 ? len : 2 * w + 1;
		warp_ksw_global(lane, len, qs, rlen, rs, s_mat, 5, 1, 5, 1, w, H, E, z, n_col, &cells);
		if (lane == 0) {
			u32 *cig = a.cig + tk.cig_off;
			int n = ksw_backtrack(z, n_col, rlen, len, w, cig), shift = 0;
			if ((cig[n - 1] & 0xf) == 1) cig[n - 1] = cig[n - 1] >> 4 << 4 | 3;   /* an insertion at either end becomes a soft clip */
			if ((cig[0] & 0xf) == 1) cig[0] = cig[0] >> 4 << 4 | 3;
			if ((cig[n - 1] & 0xf) == 2) --n;                                       /* a deletion at the end is dropped */
			if ((cig[0] & 0xf) == 2) {                                              /* one at the start moves the position */
				shift = (int)(cig[0] >> 4);
				--n;
				for (int k = 0; k < n; ++k) cig[k] = cig[k + 1];
			}
			for (int k = 0; k < n; ++k) cig[k] = se_cigar16(cig[k] & 0xf, cig[k] >> 4);
			a.ncig[t] = n; a.tshift[t] = shift;
			++n_run;
		}
		__syncwarp();
	}
	if (lane == 0 && cells) { atomicAdd(a.cells, cells); atomicAdd(a.n_run, n_run); }
}


/* S4 (see the file comment).  rec[r].len_a / len_b come from pass 0; pass 1 fills rec[r].off and flags and writes the text */
__global__ void k_se_text(DevIndex ix, SeArgs a, int write)
{
	for (int r = blockIdx.x * blockDim.x + threadIdx.x; r < a.n_reads; r += gridDim.x * blockDim.x) {
		const bwag_se_read_t p = a.reads[r];
		const i64 o0 = write ? a.tbeg[r] : 0;
		SeOut o = { write ? a.text + o0 : 0, 0 };
		const uint8_t *read = a.codes + a.off[r];
		const int full_len = (int)(a.off[r + 1] - a.off[r]), len = p.len;
		const bool mapped = a.mapped[r] != 0;
		const int strand = mapped ? a.strand[r] : 0;
		i64 len_a;
		if (mapped) {
			const int t = a.main_task[r];
			const u32 *cig = t >= 0 ? a.cig + a.tasks[t].cig_off : 0;
			const int n_cigar = t >= 0 ? a.ncig[t] : 0;
			const i64 pos = a.pos[r] + (t >= 0 ? a.tshift[t] : 0);
			const SeCig ec = se_corrected(cig, n_cigar, len, full_len, strand);
			i64 x = pos;   /* pos_end over the corrected CIGAR; without one (untrimmed, ungapped) the full length */
			if (ec.n) { for (int k = 0; k < ec.n; ++k) { const u32 cv = ec.at(k); if (se_op(cv) == 0 || se_op(cv) == 2) x += se_len(cv); } }
			else x += full_len;
			int seqid, flag = 0;
			const int nn = se_cnt_ambi(a, pos, (int)(x - pos), &seqid);
			if (pos + (x - pos) - a.ctg.off[seqid] > a.ctg.len[seqid]) flag |= 4;   /* bridges two adjacent contigs */
			if (strand) flag |= 16;
			o.c('\t'); o.d(flag); o.c('\t');
			o.s(a.ctg.names + a.ctg.name_off[seqid], a.ctg.name_off[seqid + 1] - a.ctg.name_off[seqid]);
			o.c('\t'); o.d((int)(pos - a.ctg.off[seqid] + 1)); o.c('\t'); o.d(p.mapq); o.c('\t');
			if (ec.n) for (int k = 0; k < ec.n; ++k) { const u32 cv = ec.at(k); o.d(se_len(cv)); o.c("MIDS"[se_op(cv)]); }
			else { o.d(full_len); o.c('M'); }
			o.s("\t*\t0\t0\t");
			if (!strand) for (int i = 0; i < full_len; ++i) o.c("ACGTN\0"[read[i]]);
			else for (int i = full_len - 1; i >= 0; --i) o.c("TGCAN\0"[read[i]]);
			o.c('\t');
			len_a = o.n;
			if (a.l_rg) { o.s("\tRG:Z:"); o.s(a.rg, a.l_rg); }
			if (p.l_bc) { o.s("\tBC:Z:"); o.s(a.bc + p.bc_off, p.l_bc); }
			if (p.clip_len < full_len) { o.s("\tXC:i:"); o.d(p.clip_len); }
			/* MD and NM on the searched bases, before the trimming correction, in one walk: NM is printed first, so pass 0 walks into a
			 * counter and keeps NM for pass 1, which walks once more, into the text */
			const SeRead q = { read, len, strand != 0, (a.mode & BWAG_SE_COMPREAD) != 0 };
			SeOut md_count = { 0, 0 };
			const int nm = write ? a.nm[r] : se_md(ix, a.ctg.l_pac, cig, n_cigar, q, pos, &md_count);
			if (!write) a.nm[r] = nm;
			char xt = "NURM"[p.type & 3];
			if (nn > 10) xt = 'N';
			o.s("\tXT:A:"); o.c(xt);
			o.s((a.mode & BWAG_SE_COMPREAD) ? "\tNM:i:" : "\tCM:i:"); o.d(nm & 0xfff);
			if (nn) { o.s("\tXN:i:"); o.d(nn); }
			o.s("\tX0:i:"); o.d((int)p.c1);
			if ((int)p.c1 <= a.max_top2) { o.s("\tX1:i:"); o.d((int)p.c2); }
			o.s("\tXM:i:"); o.d(p.n_mm); o.s("\tXO:i:"); o.d(p.n_gapo); o.s("\tXG:i:"); o.d(p.n_gapo + p.n_gape);
			o.s("\tMD:Z:");
			if (write) se_md(ix, a.ctg.l_pac, cig, n_cigar, q, pos, &o);
			else o.n += md_count.n;
			/* XA: the candidates kept, refined if gapped; pos_end_multi with the corrected (full) length */
			bool any = false;
			for (int k = 0; k < p.n_multi; ++k) {
				const i64 s = p.multi_beg + k;
				if (!a.mkeep[s]) continue;
				if (!any) { o.s("\tXA:Z:"); any = true; }
				const int mt = a.multi_task[s];
				const u32 *mc = mt >= 0 ? a.cig + a.tasks[mt].cig_off : 0;
				const int mn = mt >= 0 ? a.ncig[mt] & 0x7fff : 0;   /* bwt_multi1_t keeps n_cigar in 15 bits */
				const i64 mp = a.mpos[s] + (mt >= 0 ? a.tshift[mt] : 0);
				i64 e = mp;
				if (mc) { for (int j = 0; j < mn; ++j) { const int op = se_op(mc[j]); if (op == 0 || op == 2) e += se_len(mc[j]); } }
				else e += full_len;
				int sid;
				se_cnt_ambi(a, mp, (int)(e - mp), &sid);
				o.s(a.ctg.names + a.ctg.name_off[sid], a.ctg.name_off[sid + 1] - a.ctg.name_off[sid]);
				o.c(','); o.c(a.mstrand[s] ? '-' : '+'); o.d((int)(mp - a.ctg.off[sid] + 1)); o.c(',');
				if (mc) for (int j = 0; j < mn; ++j) { o.d(se_len(mc[j])); o.c("MIDS"[se_op(mc[j])]); }
				else { o.d(full_len); o.c('M'); }
				o.c(','); o.d((int)a.multi[s].gap + (int)a.multi[s].mm); o.c(';');
			}
		} else {
			o.s("\t4\t*\t0\t0\t*\t*\t0\t0\t");
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
