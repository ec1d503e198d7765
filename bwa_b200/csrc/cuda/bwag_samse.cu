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
#include "bwag_drv.h"
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
		int w = (int)(abs(rlen - len) * 1.5);   /* in range: rlen - len is the hit's n_del - n_ins */
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

/* ------------------------------------------------------------------------------------------------ host driver */

extern "C" int bwag_ctx_set_ambs(bwag_ctx_t *c, int n_holes, const int64_t *offset, const int32_t *len)
{
	CK(cudaSetDevice(c->device));
	const size_t bytes = 12 * (size_t)(n_holes > 0 ? n_holes : 0) + 16;   /* offsets | lengths */
	char *h = (char *)calloc(1, bytes);
	if (!h) return set_err("out of memory");
	if (n_holes > 0) { memcpy(h, offset, 8 * (size_t)n_holes); memcpy(h + 8 * (size_t)n_holes, len, 4 * (size_t)n_holes); }
	pthread_mutex_lock(&c->mu);
	if (c->ambs.p) { cudaStreamSynchronize(c->lane.stream); cudaFree(c->ambs.p); c->ambs.p = 0; c->have_ambs = 0; }
	cudaError_t e = cudaMalloc(&c->ambs.p, bytes);
	if (e == cudaSuccess) e = cudaMemcpy(c->ambs.p, h, bytes, cudaMemcpyHostToDevice);
	free(h);
	if (e != cudaSuccess) { pthread_mutex_unlock(&c->mu); return set_err("upload of the holes failed: %s", cudaGetErrorString(e)); }
	c->n_holes = n_holes > 0 ? n_holes : 0; c->have_ambs = 1;
	pthread_mutex_unlock(&c->mu);
	return 0;
}

#ifdef BWAG_CUSIM
#define SE_BUDGET ((i64)256 << 20)
#define SE_WARPS_PER_SM 1
#else
#define SE_BUDGET ((i64)4 << 30)     /* per-warp scratch of the refinement (backtrack bytes above all) */
#define SE_WARPS_PER_SM 32
#endif

/* the refinement tasks of read r (S3, P6): its chosen hit if `gapped`, then each of its XA candidates with a gap; mtask[r] and
 * mtask[n + slot] get the task or -1.  A task's CIGAR gets len + rlen + 2 words (a global alignment has at most len + rlen
 * operations); its band is max(50, 1.5 |rlen - len|) */
int se_list_read(SeList &L, const bwag_se_read_t &p, const bwag_se_hit_t *multi, int r, bool gapped, int *mtask, int n)
{
	for (int k = -1; k < p.n_multi; ++k) {
		const i64 slot = k < 0 ? -1 : p.multi_beg + k;
		int &mt = k < 0 ? mtask[r] : mtask[n + slot];
		mt = -1;
		if (k < 0 ? !gapped : !multi[slot].gap) continue;
		const int rlen = p.len + (k < 0 ? p.ref_shift : multi[slot].ref_shift);
		if (rlen < 0) return set_err("read %d of the batch: a gapped hit with %d reference bases", r, rlen);
		int w = (int)(abs(rlen - p.len) * 1.5);   /* in range: rlen - len is the hit's n_del - n_ins */
		w = w > 50 ? w : 50;
		const i64 n_col = p.len < 2 * w + 1 ? p.len : 2 * w + 1;
		mt = L.n_tasks;
		L.tasks[L.n_tasks].read = r; L.tasks[L.n_tasks].slot = (int)slot; L.tasks[L.n_tasks].cig_off = L.n_cig;
		++L.n_tasks;
		L.n_cig += (i64)p.len + rlen + 2;
		if (p.len > L.cap_q) L.cap_q = p.len;
		if (rlen > L.cap_r) L.cap_r = rlen;
		if (n_col * rlen > L.cap_z) L.cap_z = n_col * rlen;
	}
	return 0;
}

/* the arguments of S3/S4 and P6/P7 over the batch's samse buffers, the contig table and the holes */
void se_args(bwag_batch_t *b, SeArgs &a, int n_tasks, i64 nm, int mode, int max_top2, i64 l_bc, int l_rg)
{
	Lane *c = &b->lane;
	const bwag_ctx_t *pc = b->ctx;
	const int n = b->n;
	memset(&a, 0, sizeof(a));
	a.n_reads = n; a.n_multi = nm; a.n_tasks = n_tasks; a.mode = mode; a.max_top2 = max_top2;
	a.ctg = pc->tctg; a.n_holes = pc->n_holes; a.amb_off = (const i64 *)pc->ambs.p; a.amb_len = (const int *)((const char *)pc->ambs.p + 8 * (size_t)pc->n_holes);
	a.codes = (const uint8_t *)b->d_codes.p; a.off = (const i64 *)b->d_off.p;
	a.reads = (const bwag_se_read_t *)b->d_se_reads.p; a.multi = (const bwag_se_hit_t *)b->d_se_multi.p;
	a.bc = (const char *)b->d_se_bc.p; a.rg = (const char *)b->d_se_bc.p + l_bc; a.l_rg = l_rg;
	a.pos = (i64 *)b->d_se_pos.p; a.mpos = (i64 *)b->d_se_mpos.p;
	a.strand = (uint8_t *)b->d_se_flags.p; a.mapped = a.strand + n; a.mstrand = a.mapped + n; a.mkeep = a.mstrand + nm;
	a.tasks = (const SeTask *)b->d_se_tasks.p; a.main_task = (const int *)b->d_se_mtask.p; a.multi_task = a.main_task + n;
	a.cig = (u32 *)b->d_se_cig.p; a.ncig = (int *)b->d_se_ncig.p; a.tshift = a.ncig + n_tasks;
	a.next_task = &c->d_cnt->se_next; a.past_end = &c->d_cnt->se_past; a.n_run = &c->d_cnt->se_run; a.cells = &c->d_cnt->se_cells;
	a.tlen = (i64 *)b->d_se_tlen.p; a.tbeg = (const i64 *)b->d_se_tbeg.p; a.rec = (bwag_samrec_t *)b->d_se_rec.p; a.nm = (int *)b->d_se_nm.p;
}

/* the per-warp scratch of S3 and P5 in b->d_se_scratch: H/E rows, the reference window, the query (none if qseq is NULL) and the
 * backtrack bytes, for as many warps as the tasks, SE_WARPS_PER_SM per SM and SE_BUDGET allow; returns the warps, 0 on error */
i64 se_scratch(bwag_batch_t *b, int n_tasks, int cap_q, int cap_r, i64 cap_z, int **eh, uint8_t **rseq, uint8_t **qseq, uint8_t **z)
{
	const i64 per_warp = (8 * ((i64)cap_q + 2) + cap_r + (qseq ? cap_q : 0) + cap_z + 15) & ~(i64)15;
	i64 warps = (i64)b->ctx->n_sm * SE_WARPS_PER_SM;
	if (warps > n_tasks) warps = n_tasks;
	if (warps > SE_BUDGET / per_warp) warps = SE_BUDGET / per_warp;
	if (warps < 1) warps = 1;
	warps = (warps + 3) & ~(i64)3;   /* whole blocks of SE_THREADS */
	if (buf_reserve(&b->d_se_scratch, (size_t)(warps * per_warp))) return 0;
	unsigned char *sc = (unsigned char *)b->d_se_scratch.p;
	*eh = (int *)sc; sc += warps * 8 * ((i64)cap_q + 2);
	*rseq = sc; sc += warps * (i64)cap_r;
	if (qseq) { *qseq = sc; sc += warps * (i64)cap_q; }
	*z = sc;
	return warps;
}

/* S1, K2, S2 and S3, then S4 twice around a scan: every buffer is sized from the parameters or a scan's total.  The gapped hits
 * and the room of their CIGARs are listed here, from what the caller gives; the device skips those whose hit turns out unmapped
 * or leaves XA. */
extern "C" int bwag_samse(bwag_batch_t *b, const bwag_samse_par_t *par, bwag_sam_t *out, int *past_end, int64_t *n_sa, int64_t *n_glb)
{
	Lane *c = &b->lane;
	const bwag_ctx_t *pc = b->ctx;
	CK(cudaSetDevice(pc->device));
	memset(out, 0, sizeof(*out));
	*past_end = -1; *n_sa = 0; *n_glb = 0;
	if (!pc->have_ctg || !pc->have_ambs) return set_err("bwag_samse needs the contig table and the holes (bwag_ctx_set_contigs, bwag_ctx_set_ambs)");
	const int n = b->n;
	const i64 nm = par->n_multi, n_rows = (i64)n + nm;
	if (hbuf_reserve(&b->h_se_tasks, sizeof(SeTask) * ((size_t)n_rows + 1)) || hbuf_reserve(&b->h_se_mtask, 4 * ((size_t)n_rows + 1))) return 1;
	SeList L;
	L.tasks = (SeTask *)b->h_se_tasks.p;
	int *mtask = (int *)b->h_se_mtask.p;   /* [n] the chosen hit's task, then [nm] each candidate's */
	i64 n_mapped = 0;
	for (int r = 0; r < n; ++r) {
		const bwag_se_read_t &p = par->reads[r];
		if (p.len < 1 || p.len > (int)(b->h_off[r + 1] - b->h_off[r])) return set_err("read %d of the batch: %d bases searched of %lld", r, p.len, (long long)(b->h_off[r + 1] - b->h_off[r]));
		n_mapped += p.type != 0;
		if (se_list_read(L, p, par->multi, r, p.type && p.n_gapo, mtask, n)) return 1;
	}
	const int n_tasks = L.n_tasks;
	const i64 n_cig = L.n_cig;
	*n_sa = n_mapped + nm;
	const size_t l_rg = par->rg_id ? strlen(par->rg_id) : 0;
	if (buf_reserve(&b->d_se_reads, sizeof(bwag_se_read_t) * ((size_t)n + 1)) || buf_reserve(&b->d_se_multi, sizeof(bwag_se_hit_t) * ((size_t)nm + 1)) ||
	    buf_reserve(&b->d_se_bc, (size_t)par->l_bc + l_rg + 16) || buf_reserve(&b->d_se_rows, 8 * ((size_t)n_rows + 1)) ||
	    buf_reserve(&b->d_se_pos, 8 * ((size_t)n + 1)) || buf_reserve(&b->d_se_mpos, 8 * ((size_t)nm + 1)) || buf_reserve(&b->d_se_flags, 2 * (size_t)n_rows + 16) ||
	    buf_reserve(&b->d_se_tasks, sizeof(SeTask) * ((size_t)n_tasks + 1)) || buf_reserve(&b->d_se_mtask, 4 * ((size_t)n_rows + 1)) ||
	    buf_reserve(&b->d_se_cig, 4 * ((size_t)n_cig + 1)) || buf_reserve(&b->d_se_ncig, 8 * ((size_t)n_tasks + 1)) ||
	    buf_reserve(&b->d_se_tlen, 8 * ((size_t)n + 1)) || buf_reserve(&b->d_se_tbeg, 8 * ((size_t)n + 1)) || buf_reserve(&b->d_se_nm, 4 * ((size_t)n + 1)) || buf_reserve(&b->d_se_rec, sizeof(bwag_samrec_t) * ((size_t)n + 1)) ||
	    hbuf_reserve(&b->h_se_rec, sizeof(bwag_samrec_t) * ((size_t)n + 1))) return 1;
	SeArgs a;
	se_args(b, a, n_tasks, nm, par->mode, par->max_top2, par->l_bc, (int)l_rg);
	a.rows = (i64 *)b->d_se_rows.p;
	if (reset_counters(c)) return 1;
	if (n) H2D(c, b->d_se_reads.p, par->reads, sizeof(bwag_se_read_t) * (size_t)n);
	if (nm) H2D(c, b->d_se_multi.p, par->multi, sizeof(bwag_se_hit_t) * (size_t)nm);
	if (par->l_bc) H2D(c, b->d_se_bc.p, par->bc, (size_t)par->l_bc);
	if (l_rg) H2D(c, (char *)b->d_se_bc.p + par->l_bc, par->rg_id, l_rg);
	if (n_tasks) H2D(c, b->d_se_tasks.p, L.tasks, sizeof(SeTask) * (size_t)n_tasks);
	if (n_rows) H2D(c, b->d_se_mtask.p, mtask, 4 * (size_t)n_rows);
	/* S1 + K2: the rows, resolved in place; S2 */
	if (n_rows) {
		BWAG_LAUNCH(k_se_rows, fm_grid(pc, n_rows), 128, 0, c->stream, a);
		if (run_sa(b, a.rows, n_rows)) return 1;
		BWAG_LAUNCH(k_se_pos, fm_grid(pc, n), 128, 0, c->stream, a);
		CK(cudaGetLastError());
		c->st.n_launch += 3;
	}
	/* S3: persistent warps over the gapped hits, as many as the scratch budget allows */
	if (n_tasks) {
		const i64 warps = se_scratch(b, n_tasks, L.cap_q, L.cap_r, L.cap_z, &a.eh, &a.rseq, &a.qseq, &a.z);
		if (!warps) return 1;
		a.cap_q = L.cap_q; a.cap_r = L.cap_r; a.cap_z = L.cap_z;
		CK(cudaMemsetAsync(b->d_se_ncig.p, 0, 8 * (size_t)n_tasks, c->stream));
		BWAG_LAUNCH(k_se_refine, (int)(warps * 32 / SE_THREADS), SE_THREADS, 0, c->stream, c->ix, a);
		CK(cudaGetLastError());
		++c->st.n_launch;
	}
	/* S4: sizes, their scan, then the text */
	if (n) BWAG_LAUNCH(k_se_text, fm_grid(pc, n), 128, 0, c->stream, c->ix, a, 0);
	BWAG_LAUNCH(k_fm_scan64, 1, FM_SCAN_THREADS, 0, c->stream, (const i64 *)b->d_se_tlen.p, (i64)n, (i64 *)b->d_se_tbeg.p, &c->d_cnt->se_total);
	CK(cudaGetLastError());
	if (fetch_counters(c)) return 1;
	c->st.n_launch += 2;
	if (n_rows) { c->st.ms_sa += elapsed_at(c, "sa", __FILE__, __LINE__); c->st.sa_touches += c->h_cnt->sa_touches; }
	c->st.glb_cells += c->h_cnt->se_cells;
	*n_glb = (int64_t)c->h_cnt->se_run;
	if (c->h_cnt->se_past) {
		*past_end = n - c->h_cnt->se_past;
		return set_err("read %d of the batch: its gapped alignment window runs past the end of the forward strand", *past_end);
	}
	const i64 n_text = (i64)c->h_cnt->se_total;
	if (buf_reserve(&b->d_se_text, (size_t)n_text + 1) || hbuf_reserve(&b->h_se_text, (size_t)n_text + 1)) return 1;
	a.text = (char *)b->d_se_text.p;
	if (n) BWAG_LAUNCH(k_se_text, fm_grid(pc, n), 128, 0, c->stream, c->ix, a, 1);
	CK(cudaGetLastError());
	++c->st.n_launch;
	CK(cudaEventRecord(c->ev0, c->stream));
	if (n_text) D2H(c, b->h_se_text.p, b->d_se_text.p, (size_t)n_text);
	if (n) D2H(c, b->h_se_rec.p, b->d_se_rec.p, sizeof(bwag_samrec_t) * (size_t)n);
	CK(cudaEventRecord(c->ev1, c->stream));
	CK(stream_wait(c));
	c->st.ms_d2h += elapsed_at(c, "d2h", __FILE__, __LINE__);
	out->rec = (const bwag_samrec_t *)b->h_se_rec.p; out->text = (const char *)b->h_se_text.p; out->n_text = n_text;
	return 0;
}
