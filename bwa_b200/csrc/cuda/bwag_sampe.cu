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
#include "bwag_drv.h"
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

/* ------------------------------------------------------------------------------------------------ host driver */

/* P1/P2: K2 resolves the rows in place, k_pe_pos applies bwa_sa2pos twice per row */
extern "C" int bwag_pe_sa2pos(bwag_batch_t *b, int64_t n_rows, const uint64_t *rows, const int32_t *ref_len, int64_t *pos, uint8_t *strand)
{
	Lane *c = &b->lane;
	CK(cudaSetDevice(b->ctx->device));
	if (n_rows <= 0) return 0;
	const size_t n = (size_t)n_rows;
	if (buf_reserve(&b->d_se_rows, 8 * n) || buf_reserve(&b->d_pe_rlen, 8 * n) || buf_reserve(&b->d_se_pos, 16 * n) || buf_reserve(&b->d_se_flags, 2 * n + 16) ||
	    hbuf_reserve(&b->h_pe_pos, 18 * n + 16)) return 1;
	PePosArgs a;
	a.n = n_rows; a.l_pac = (i64)c->ix.l_pac; a.rows = (const i64 *)b->d_se_rows.p; a.ref_len = (const int *)b->d_pe_rlen.p;
	a.pos = (i64 *)b->d_se_pos.p; a.strand = (uint8_t *)b->d_se_flags.p;
	if (reset_counters(c)) return 1;
	H2D(c, b->d_se_rows.p, rows, 8 * n);
	H2D(c, b->d_pe_rlen.p, ref_len, 8 * n);
	if (run_sa(b, (i64 *)b->d_se_rows.p, n_rows)) return 1;
	BWAG_LAUNCH(k_pe_pos, fm_grid(b->ctx, n_rows), 128, 0, c->stream, a);
	CK(cudaGetLastError());
	c->st.n_launch += 2;
	char *h = (char *)b->h_pe_pos.p;
	D2H(c, h, b->d_se_pos.p, 16 * n);
	D2H(c, h + 16 * n, b->d_se_flags.p, 2 * n);
	CK(stream_wait(c));
	c->st.ms_sa += elapsed_at(c, "sa", __FILE__, __LINE__);
	memcpy(pos, h, 16 * n); memcpy(strand, h + 16 * n, 2 * n);
	return 0;
}

/* P5: the global alignments of the accepted local ones, one warp each, as many warps as the scratch budget allows */
extern "C" int bwag_pe_global(bwag_batch_t *b, int n_tasks, const bwag_pe_gtask_t *tasks, const uint8_t *pool, size_t pool_bytes, const bwag_pe_gres_t **res, const uint32_t **cig)
{
	Lane *c = &b->lane;
	CK(cudaSetDevice(b->ctx->device));
	*res = 0; *cig = 0;
	if (n_tasks <= 0) return 0;
	int cap_q = 1, cap_r = 1;
	i64 cap_z = 1, n_cig = 0;
	if (hbuf_reserve(&b->h_pe_gres, sizeof(bwag_pe_gres_t) * (size_t)n_tasks)) return 1;
	bwag_pe_gres_t *hr = (bwag_pe_gres_t *)b->h_pe_gres.p;
	for (int t = 0; t < n_tasks; ++t) {
		const bwag_pe_gtask_t &tk = tasks[t];
		if (tk.qlen < 1 || tk.tlen < 1 || tk.q_beg < 0 || tk.q_beg + tk.qlen > (i64)pool_bytes || tk.t_beg < 0 || tk.t_beg + tk.tlen > (i64)c->ix.l_pac)
			return set_err("mate-rescue alignment %d: query [%lld, +%d) or target [%lld, +%d) out of range", t, (long long)tk.q_beg, tk.qlen, (long long)tk.t_beg, tk.tlen);
		const int n_col = tk.qlen < 101 ? tk.qlen : 101;
		hr[t].score = 0; hr[t].n_cigar = 0; hr[t].cig_off = n_cig;
		n_cig += (i64)tk.qlen + tk.tlen + 2;
		if (tk.qlen > cap_q) cap_q = tk.qlen;
		if (tk.tlen > cap_r) cap_r = tk.tlen;
		if ((i64)n_col * tk.tlen > cap_z) cap_z = (i64)n_col * tk.tlen;
	}
	if (buf_reserve(&b->d_pe_gtasks, sizeof(bwag_pe_gtask_t) * (size_t)n_tasks) || buf_reserve(&b->d_pe_gres, sizeof(bwag_pe_gres_t) * (size_t)n_tasks) ||
	    buf_reserve(&b->d_pe_gcig, 4 * (size_t)n_cig) || buf_reserve(&b->d_pe_pool, pool_bytes + 16) || hbuf_reserve(&b->h_pe_gcig, 4 * (size_t)n_cig)) return 1;
	PeGlbArgs a;
	const i64 warps = se_scratch(b, n_tasks, cap_q, cap_r, cap_z, &a.eh, &a.rseq, 0, &a.z);
	if (!warps) return 1;
	a.n_tasks = n_tasks; a.tasks = (const bwag_pe_gtask_t *)b->d_pe_gtasks.p; a.res = (bwag_pe_gres_t *)b->d_pe_gres.p; a.cig = (u32 *)b->d_pe_gcig.p;
	a.pool = (const uint8_t *)b->d_pe_pool.p;
	a.cap_q = cap_q; a.cap_r = cap_r; a.cap_z = cap_z;
	a.next_task = &c->d_cnt->se_next; a.cells = &c->d_cnt->se_cells;
	if (reset_counters(c)) return 1;
	H2D(c, b->d_pe_gtasks.p, tasks, sizeof(bwag_pe_gtask_t) * (size_t)n_tasks);
	H2D(c, b->d_pe_gres.p, hr, sizeof(bwag_pe_gres_t) * (size_t)n_tasks);
	H2D(c, b->d_pe_pool.p, pool, pool_bytes);
	BWAG_LAUNCH(k_pe_global, (int)(warps * 32 / SE_THREADS), SE_THREADS, 0, c->stream, c->ix, a);
	CK(cudaGetLastError());
	++c->st.n_launch;
	D2H(c, b->h_pe_gres.p, b->d_pe_gres.p, sizeof(bwag_pe_gres_t) * (size_t)n_tasks);
	D2H(c, b->h_pe_gcig.p, b->d_pe_gcig.p, 4 * (size_t)n_cig);
	if (fetch_counters(c)) return 1;
	c->st.glb_cells += c->h_cnt->se_cells;
	*res = (const bwag_pe_gres_t *)b->h_pe_gres.p; *cig = (const uint32_t *)b->h_pe_gcig.p;
	return 0;
}

/* P6 (samse's S3 on the caller's positions) and P7, around a scan */
extern "C" int bwag_sampe(bwag_batch_t *b, const bwag_sampe_par_t *par, bwag_sam_t *out, int *past_end, int64_t *n_glb)
{
	Lane *c = &b->lane;
	const bwag_ctx_t *pc = b->ctx;
	CK(cudaSetDevice(pc->device));
	memset(out, 0, sizeof(*out));
	*past_end = -1; *n_glb = 0;
	if (!pc->have_ctg || !pc->have_ambs) return set_err("bwag_sampe needs the contig table and the holes (bwag_ctx_set_contigs, bwag_ctx_set_ambs)");
	const int n = b->n;
	if (n & 1) return set_err("bwag_sampe: a batch of %d reads is not a batch of pairs", n);
	const i64 nm = par->n_multi, n_rows = (i64)n + nm;
	if (hbuf_reserve(&b->h_se_tasks, sizeof(SeTask) * ((size_t)n_rows + 1)) || hbuf_reserve(&b->h_se_mtask, 4 * ((size_t)n_rows + 1))) return 1;
	SeList L;
	L.tasks = (SeTask *)b->h_se_tasks.p;
	int *mtask = (int *)b->h_se_mtask.p;
	int n_tasks1 = 0;   /* the tasks of end 1 come first: each end's rseq is complemented as its own .sai says */
	for (int e = 0; e < 2; ++e) for (int r = e; r < n; r += 2) {
		if (e == 1 && r == 1) n_tasks1 = L.n_tasks;
		const bwag_se_read_t &p = par->reads[r];
		if (p.len < 1 || p.len > (int)(b->h_off[r + 1] - b->h_off[r])) return set_err("read %d of the batch: %d bases searched of %lld", r, p.len, (long long)(b->h_off[r + 1] - b->h_off[r]));
		if (se_list_read(L, p, par->multi, r, (p.type == 1 || p.type == 2) && p.n_gapo, mtask, n)) return 1;
	}
	const int n_tasks = L.n_tasks;
	const i64 cig_base = L.n_cig, n_cig = cig_base + par->n_cig;   /* the mate-rescued CIGARs follow the refinement's */
	const size_t l_rg = par->rg_id ? strlen(par->rg_id) : 0;
	if (buf_reserve(&b->d_se_reads, sizeof(bwag_se_read_t) * ((size_t)n + 1)) || buf_reserve(&b->d_se_multi, sizeof(bwag_se_hit_t) * ((size_t)nm + 1)) ||
	    buf_reserve(&b->d_pe_reads, sizeof(bwag_pe_read_t) * ((size_t)n + 1)) ||
	    buf_reserve(&b->d_se_bc, (size_t)par->l_bc + l_rg + 16) ||
	    buf_reserve(&b->d_se_pos, 8 * ((size_t)n + 1)) || buf_reserve(&b->d_se_mpos, 8 * ((size_t)nm + 1)) || buf_reserve(&b->d_se_flags, 2 * (size_t)n_rows + 16) ||
	    buf_reserve(&b->d_se_tasks, sizeof(SeTask) * ((size_t)n_tasks + 1)) || buf_reserve(&b->d_se_mtask, 4 * ((size_t)n_rows + 1)) ||
	    buf_reserve(&b->d_se_cig, 4 * ((size_t)n_cig + 1)) || buf_reserve(&b->d_se_ncig, 8 * ((size_t)n_tasks + 1)) ||
	    buf_reserve(&b->d_se_tlen, 8 * ((size_t)n + 1)) || buf_reserve(&b->d_se_tbeg, 8 * ((size_t)n + 1)) || buf_reserve(&b->d_se_nm, 4 * ((size_t)n + 1)) || buf_reserve(&b->d_se_rec, sizeof(bwag_samrec_t) * ((size_t)n + 1)) ||
	    hbuf_reserve(&b->h_se_rec, sizeof(bwag_samrec_t) * ((size_t)n + 1)) || hbuf_reserve(&b->h_pe_gres, sizeof(bwag_pe_read_t) * ((size_t)n + 1))) return 1;
	bwag_pe_read_t *pe = (bwag_pe_read_t *)b->h_pe_gres.p;   /* the caller's, with the rescued CIGARs moved behind the refinement's */
	for (int r = 0; r < n; ++r) { pe[r] = par->pe[r]; if (par->reads[r].type == 3) pe[r].cig_off += cig_base; }
	SeArgs a;
	se_args(b, a, n_tasks, nm, par->mode, par->max_top2, par->l_bc, (int)l_rg);
	if (reset_counters(c)) return 1;
	{   /* mapped[] (type 1 or 2: refined when gapped) and mkeep[] (every candidate given), in pinned memory for the copy */
		if (hbuf_reserve(&b->h_pe_pos, (size_t)n + (size_t)nm + 16)) return 1;
		uint8_t *f = (uint8_t *)b->h_pe_pos.p;
		for (int r = 0; r < n; ++r) f[r] = par->reads[r].type == 1 || par->reads[r].type == 2;
		memset(f + n, 1, (size_t)nm);
		H2D(c, a.mapped, f, (size_t)n);
		if (nm) H2D(c, a.mkeep, f + n, (size_t)nm);
	}
	H2D(c, b->d_se_reads.p, par->reads, sizeof(bwag_se_read_t) * (size_t)n);
	H2D(c, b->d_pe_reads.p, pe, sizeof(bwag_pe_read_t) * (size_t)n);
	H2D(c, a.pos, par->pos, 8 * (size_t)n);
	H2D(c, a.strand, par->strand, (size_t)n);
	if (nm) { H2D(c, b->d_se_multi.p, par->multi, sizeof(bwag_se_hit_t) * (size_t)nm); H2D(c, a.mpos, par->mpos, 8 * (size_t)nm); H2D(c, a.mstrand, par->mstrand, (size_t)nm); }
	if (par->n_cig) H2D(c, a.cig + cig_base, par->cig, 4 * (size_t)par->n_cig);
	if (par->l_bc) H2D(c, b->d_se_bc.p, par->bc, (size_t)par->l_bc);
	if (l_rg) H2D(c, (char *)b->d_se_bc.p + par->l_bc, par->rg_id, l_rg);
	if (n_tasks) H2D(c, b->d_se_tasks.p, L.tasks, sizeof(SeTask) * (size_t)n_tasks);
	H2D(c, b->d_se_mtask.p, mtask, 4 * (size_t)n_rows);
	if (n_tasks) {
		const i64 warps = se_scratch(b, n_tasks, L.cap_q, L.cap_r, L.cap_z, &a.eh, &a.rseq, &a.qseq, &a.z);
		if (!warps) return 1;
		a.cap_q = L.cap_q; a.cap_r = L.cap_r; a.cap_z = L.cap_z;
		CK(cudaMemsetAsync(b->d_se_ncig.p, 0, 8 * (size_t)n_tasks, c->stream));
		for (int e = 0; e < 2; ++e) {   /* S3 once per end, with that end's COMPREAD bit */
			const int t0 = e ? n_tasks1 : 0, nt = e ? n_tasks - n_tasks1 : n_tasks1;
			if (!nt) continue;
			SeArgs ae = a;
			ae.tasks = a.tasks + t0; ae.ncig = a.ncig + t0; ae.tshift = a.tshift + t0; ae.n_tasks = nt;
			ae.mode = par->comp[e] ? BWAG_SE_COMPREAD : 0;
			CK(cudaMemsetAsync(&c->d_cnt->se_next, 0, sizeof(int), c->stream));
			BWAG_LAUNCH(k_se_refine, (int)(warps * 32 / SE_THREADS), SE_THREADS, 0, c->stream, c->ix, ae);
			CK(cudaGetLastError());
			++c->st.n_launch;
		}
	}
	const bwag_pe_read_t *d_pe = (const bwag_pe_read_t *)b->d_pe_reads.p;
	BWAG_LAUNCH(k_pe_text, fm_grid(pc, n), 128, 0, c->stream, c->ix, a, d_pe, 0);
	BWAG_LAUNCH(k_fm_scan64, 1, FM_SCAN_THREADS, 0, c->stream, (const i64 *)b->d_se_tlen.p, (i64)n, (i64 *)b->d_se_tbeg.p, &c->d_cnt->se_total);
	CK(cudaGetLastError());
	if (fetch_counters(c)) return 1;
	c->st.n_launch += 2;
	c->st.glb_cells += c->h_cnt->se_cells;
	*n_glb = (int64_t)c->h_cnt->se_run;
	if (c->h_cnt->se_past) {
		*past_end = n - c->h_cnt->se_past;
		return set_err("read %d of the batch: its gapped alignment window runs past the end of the forward strand", *past_end);
	}
	const i64 n_text = (i64)c->h_cnt->se_total;
	if (buf_reserve(&b->d_se_text, (size_t)n_text + 1) || hbuf_reserve(&b->h_se_text, (size_t)n_text + 1)) return 1;
	a.text = (char *)b->d_se_text.p;
	BWAG_LAUNCH(k_pe_text, fm_grid(pc, n), 128, 0, c->stream, c->ix, a, d_pe, 1);
	CK(cudaGetLastError());
	++c->st.n_launch;
	CK(cudaEventRecord(c->ev0, c->stream));
	if (n_text) D2H(c, b->h_se_text.p, b->d_se_text.p, (size_t)n_text);
	D2H(c, b->h_se_rec.p, b->d_se_rec.p, sizeof(bwag_samrec_t) * (size_t)n);
	CK(cudaEventRecord(c->ev1, c->stream));
	CK(stream_wait(c));
	c->st.ms_d2h += elapsed_at(c, "d2h", __FILE__, __LINE__);
	out->rec = (const bwag_samrec_t *)b->h_se_rec.p; out->text = (const char *)b->h_se_text.p; out->n_text = n_text;
	return 0;
}
