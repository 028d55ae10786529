// Report writer on the device: one batch's alignment results + the FASTA / FASTQ text of its reads -> the bytes the reference's
// report stage writes for that batch (aligned.sam body rows, tabular or pairwise aligned.blast rows, aligned / other / aligned_denovo
// reads).
//   SAM rows      ReportSam::append (src/sortmerna/report_sam.cpp:64-152)
//   BLAST rows    ReportBlast::append, tabular (report_blast.cpp:99-126, 260-346) and pairwise (-blast 0, report_blast.cpp:136-251)
//   read files    ReportFastx / ReportFxOther / ReportDenovo::append + ReportFxBase::write_a_read (report_fastx.cpp:56-140,
//                 report_fx_other.cpp:50-120, report_denovo.cpp:57-130, report_fx_base.cpp:176-181), routing of output.cpp:117-142
// Layout of the text: the newline index / line classification / scans of smr_decode.cuh, then one thread per record (rpt_records_kernel).
// Every output is made in two passes: a size pass (bytes of every row / record), an exclusive scan (cub) into offsets, a write pass.
// SAM and BLAST rows are ordered (index, part) group first, then read, then alignment slot (output.cpp:196-237) by a stable radix sort
// of the live alignment slots on their group.  SEQ and QUAL of a SAM row, the columns of a pairwise BLAST block and the records of the
// read files are written by a whole warp, so a 30 kb read is not serialised on one thread; the short fields are printed by one lane
// with smr_fmt.h.
#pragma once
#include <cstdint>

#include <cub/cub.cuh>

#include "../../include/smr_b200.h"
#include "smr_decode.cuh"
#include "smr_fmt.h"

namespace smr {

// one record of the reads text
struct RptRec {
  uint64_t hdr;          // offset of the header line
  uint64_t qual;         // FASTQ: offset of the quality line
  uint32_t hdr_len;      // header without trailing white space (Readfeed right-trims every line, readfeed.cpp:579-582)
  uint32_t name_beg, name_len;   // Read::getSeqId (read.cpp:371-377): up to the first space, leading '>' / '@' removed
  uint32_t line, next;   // line of the header; line of the next record's header (or the number of lines)
  uint32_t seq_len, qual_len;
  uint32_t verbatim;     // FASTQ record already in output form (header\nseq\n+\nqual\n): written as one copy
};

// one loaded (index, part): what its rows print
struct RptGroup {
  const char* names;          // reference ids, concatenated
  const uint64_t* name_off;   // [nref + 1]
  const double* evalue;       // [65536] E-value of each score1 (host-computed, report_blast.cpp:121-126)
  const uint32_t* bits;       // [65536] bit score of each score1 (report_blast.cpp:117-119)
  uint32_t nref, index_num, part;
  uint32_t ref_base;          // the references of the groups before: BAM's refID of reference ref_num is ref_base + ref_num
  const uint8_t* refseq;      // the part's resident reference sequences (DevIndex::refseq, 0..4): pairwise BLAST prints them
  const uint32_t* ref_off;    // [nref + 1]
};

// route flags of a read: the read files it goes to, and for each of them (kind s = 0 aligned, 1 other, 2 denovo) the file among the
// kind's num_out in 2 bits from kRptFileShift + 2 * s
enum : uint32_t { kRptAligned = 1, kRptOther = 2, kRptDenovo = 4, kRptSkip = 8, kRptFileShift = 8 };
enum : uint32_t { kRptErrLen = 1, kRptErrGroup = 2, kRptErrRef = 4, kRptErrQual = 8, kRptErrCigar = 16, kRptErrSpan = 32 };
// what BAM cannot hold (the BAM writer also names the first such read)
enum : uint32_t { kRptErrBamName = 64, kRptErrBamQualLen = 128, kRptErrBamQualByte = 256 };
enum : uint32_t { kColCigar = 1, kColQcov = 2, kColQstrand = 3 };

struct RptArgs {
  const uint8_t* text; uint64_t nbytes;
  const uint64_t* nl; const uint32_t* spos; uint32_t nlines, fastq;
  const RptRec* rec; uint32_t nreads, slots;
  // the alignment slots: strided (aln_off null), read r's alignment k at r * slots + k, nslots = nreads * slots; packed, at
  // aln_off[r] + k, nslots = the sum of n_align, slot_read[i] = the read of slot i
  uint64_t nslots; const uint32_t* aln_off; const uint32_t* slot_read;
  const smr_read_result* res; const smr_aln* aln; const uint32_t* cigar; uint64_t cigar_words; const smr_aln_stats* st;
  const RptGroup* grp; uint32_t ngroups;
  uint32_t cols[4], ncols;
  double min_id, min_cov;
  uint32_t paired_in, paired_out, denovo;
  uint32_t mates;     // records 2k and 2k+1 are mates from two files
  uint32_t out2, num_out;   // -out2; files per kind of read file: 1, 2 (-out2 or -sout) or 4 (both)
  uint32_t fx_mask;   // the read files asked for (kRptAligned | kRptOther | kRptDenovo)
  uint32_t* err;
};

__device__ __forceinline__ uint64_t rpt_slot(const RptArgs& a, uint32_t r, uint32_t k) { return a.aln_off ? (uint64_t)a.aln_off[r] + k : (uint64_t)r * a.slots + k; }
__device__ __forceinline__ uint32_t rpt_read_of(const RptArgs& a, uint64_t i) { return a.aln_off ? a.slot_read[i] : (uint32_t)(i / a.slots); }

// packed results: slot_read[aln_off[r] + k] = r for every stored alignment k of read r
__global__ void rpt_slot_read_kernel(const smr_read_result* __restrict__ res, uint32_t nreads, const uint32_t* __restrict__ aln_off,
                                     uint32_t* __restrict__ slot_read) {
  for (uint32_t r = blockIdx.x * blockDim.x + threadIdx.x; r < nreads; r += gridDim.x * blockDim.x)
    for (uint32_t k = 0, n = res[r].n_align; k < n; ++k) slot_read[aln_off[r] + k] = r;
}
// n_align of every read, and a 0 at [nreads]: scanned into aln_off
__global__ void rpt_counts_kernel(const smr_read_result* __restrict__ res, uint32_t nreads, uint32_t* __restrict__ cnt) {
  for (uint32_t r = blockIdx.x * blockDim.x + threadIdx.x; r <= nreads; r += gridDim.x * blockDim.x) cnt[r] = r < nreads ? res[r].n_align : 0;
}

__device__ __forceinline__ uint64_t rpt_line_beg(const uint64_t* nl, uint32_t i) { return i ? nl[i - 1] + 1 : 0; }
__device__ __forceinline__ bool rpt_space(uint8_t c) { return c == ' ' || (c >= '\t' && c <= '\r'); }

// headers: rec_line[rec_idx[i]] = i
__global__ void rpt_header_lines_kernel(const uint32_t* __restrict__ is_hdr, const uint32_t* __restrict__ rec_idx, uint32_t nlines,
                                        uint32_t* __restrict__ rec_line) {
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < nlines; i += gridDim.x * blockDim.x)
    if (is_hdr[i]) rec_line[rec_idx[i]] = i;
}

__global__ void rpt_records_kernel(RptArgs a, const uint32_t* __restrict__ rec_line, RptRec* __restrict__ out) {
  for (uint32_t r = blockIdx.x * blockDim.x + threadIdx.x; r < a.nreads; r += gridDim.x * blockDim.x) {
    RptRec o{};
    o.line = rec_line[r];
    o.next = r + 1 < a.nreads ? rec_line[r + 1] : a.nlines;
    const uint64_t s = rpt_line_beg(a.nl, o.line);
    uint64_t e = a.nl[o.line];
    while (e > s && rpt_space(a.text[e - 1])) --e;
    o.hdr = s; o.hdr_len = (uint32_t)(e - s);
    uint32_t sp = 0;
    while (sp < o.hdr_len && a.text[s + sp] != ' ') ++sp;
    uint32_t nb = 0;
    while (nb < sp && (a.text[s + nb] == '>' || a.text[s + nb] == '@')) ++nb;
    o.name_beg = nb; o.name_len = sp - nb;
    o.seq_len = a.spos[o.next] - a.spos[o.line];
    if (a.fastq) {
      if (o.line + 3 >= a.nlines) { atomicOr(a.err, kRptErrQual); out[r] = o; continue; }
      const uint64_t qs = rpt_line_beg(a.nl, o.line + 3);
      uint64_t qe = a.nl[o.line + 3];
      while (qe > qs && rpt_space(a.text[qe - 1])) --qe;
      o.qual = qs; o.qual_len = (uint32_t)(qe - qs);
      const uint64_t out_len = (uint64_t)o.hdr_len + o.seq_len + o.qual_len + 5;
      o.verbatim = a.nl[o.line + 3] < a.nbytes && a.nl[o.line + 3] + 1 - s == out_len;   // no CR, no trailing blanks, bare '+'
    }
    out[r] = o;
  }
}

// counting / writing output cursor: p == nullptr counts only
struct RptSink {
  char* p; uint64_t n;
  __device__ void c(char x) { if (p) p[n] = x; ++n; }
  __device__ void s(const char* x, uint32_t k) { if (p) for (uint32_t i = 0; i < k; ++i) p[n + i] = x[i]; n += k; }
  __device__ void u(uint64_t v) { char t[24]; s(t, (uint32_t)fmt::put_u64(t, v)); }
  __device__ void i(int64_t v) { char t[24]; s(t, (uint32_t)fmt::put_i64(t, v)); }
  __device__ void g3(double v) { char t[24]; s(t, (uint32_t)fmt::fmt_g3(v, t)); }
};

__device__ __forceinline__ uint32_t rpt_group_of(const RptArgs& a, const smr_aln& al) {
  for (uint32_t g = 0; g < a.ngroups; ++g)
    if (a.grp[g].index_num == al.index_num && a.grp[g].part == al.part) return g;
  return a.ngroups;
}

// the soft clips of report_sam.cpp:99-116 / report_blast.cpp:318-337: the leading one is written when it is not 0, the trailing
// one when it is above 0
__device__ __forceinline__ int64_t rpt_clip_lead(const smr_aln& al) { return al.read_begin1; }
__device__ __forceinline__ int64_t rpt_clip_trail(const smr_aln& al, uint32_t read_len) { return (int64_t)read_len - al.read_end1 - 1; }

// CIGAR with the soft clips
__device__ void rpt_cigar(RptSink& o, const RptArgs& a, const smr_aln& al, uint32_t read_len) {
  if (rpt_clip_lead(al) != 0) { o.i(rpt_clip_lead(al)); o.c('S'); }
  if ((uint64_t)al.cigar_off + al.cigar_len > a.cigar_words) { atomicOr(a.err, kRptErrCigar); return; }
  for (uint32_t c = 0; c < al.cigar_len; ++c) {
    const uint32_t w = a.cigar[al.cigar_off + c], op = w & 0xF;
    o.u(w >> 4);
    o.c(op == 0 ? 'M' : op == 1 ? 'I' : 'D');
  }
  const int64_t end_mask = rpt_clip_trail(al, read_len);
  if (end_mask > 0) { o.i(end_mask); o.c('S'); }
}

// QNAME: Read::getSeqId of the record's header
__device__ __forceinline__ void rpt_qname(RptSink& o, const RptArgs& a, const RptRec& rc) { o.s((const char*)a.text + rc.hdr + rc.name_beg, rc.name_len); }

__device__ __forceinline__ void rpt_ref_name(RptSink& o, const RptArgs& a, const RptGroup& g, uint32_t ref_num) {
  if (ref_num >= g.nref) { atomicOr(a.err, kRptErrRef); return; }
  const uint64_t b = g.name_off[ref_num];
  o.s(g.names + b, (uint32_t)(g.name_off[ref_num + 1] - b));
}

// The class of one stored alignment in denovo_stats_run (processor.cpp:329-357), as hostio.denovo_classes: 0 c_yid_ycov, 1 n_yid_ncov,
// 2 n_nid_ycov, 3 n_denovo.  %id from n_match_denovo; both rounded with floor(x * 1000 + 0.5) / 1000.0, no FMA: the host rounds twice.
enum : uint32_t { kDnYidYcov = 0, kDnYidNcov = 1, kDnNidYcov = 2, kDnDenovo = 3 };
__device__ __forceinline__ uint32_t denovo_class(const smr_aln& al, const smr_aln_stats& st, double min_id, double min_cov) {
  const double id = (double)st.n_match_denovo / (double)(st.n_miss + st.n_gap + st.n_match);
  const int32_t span = al.read_end1 - al.read_begin1 + 1;
  const double cov = (double)(span < 0 ? -span : span) / (double)al.readlen;
  const bool is_id = floor(__dadd_rn(__dmul_rn(id, 1000.0), 0.5)) / 1000.0 >= min_id;
  const bool is_cov = floor(__dadd_rn(__dmul_rn(cov, 1000.0), 0.5)) / 1000.0 >= min_cov;
  return is_id && is_cov ? kDnYidYcov : is_id ? kDnYidNcov : is_cov ? kDnNidYcov : kDnDenovo;
}

// per read: routing to aligned / other / aligned_denovo and the skip of empty reads (output.cpp:117-142)
__device__ bool rpt_is_denovo(const RptArgs& a, uint32_t r) {   // n_denovo > 0 and the other three counters 0
  const uint32_t n = a.res[r].n_align;
  if (n == 0) return false;
  for (uint32_t k = 0; k < n; ++k)
    if (denovo_class(a.aln[rpt_slot(a, r, k)], a.st[rpt_slot(a, r, k)], a.min_id, a.min_cov) != kDnDenovo) return false;
  return true;
}

// The file of mate i (0 / 1) of a pair among the num_out of its kind, -1 = not written; h / hm: this read / its mate aligned;
// d / dm: denovo.  Restatements of the paired branches at -threads 1 (id 0); num_out 4 means -out2 and -sout, which exclude
// paired_in / paired_out (ReportFxBase::validate_out_type).
//   aligned  ReportFastx::append (report_fastx.cpp:71-133)
__device__ int rpt_file_aligned(const RptArgs& a, uint32_t i, bool h, bool hm) {
  const bool both = h && hm;
  if (!h && !hm) return -1;
  if (a.num_out == 1) return (a.paired_out ? both : (a.paired_in || h)) ? 0 : -1;
  if (a.num_out == 2 && a.out2) return (a.paired_out ? both : (a.paired_in || h)) ? (int)i : -1;   // paired_out: 'break' when not both
  if (a.num_out == 2) return both ? 0 : h ? 1 : -1;                                               // -sout: paired, singleton
  return both ? (int)i : h ? (int)i + 2 : -1;
}
//   other    ReportFxOther::append (report_fx_other.cpp:52-113)
__device__ int rpt_file_other(const RptArgs& a, uint32_t i, bool h, bool hm) {
  const bool any = h || hm;
  if (h && hm) return -1;
  if (a.num_out == 1) return (a.paired_in ? !any : (a.paired_out || !h)) ? 0 : -1;
  if (a.num_out == 2 && a.out2) return (a.paired_in ? !any : (a.paired_out || !h)) ? (int)i : -1;   // paired_in: 'break' when any
  if (a.num_out == 2) return !any ? 0 : !h ? 1 : -1;
  return !any ? (int)i : !h ? (int)i + 2 : -1;
}
//   denovo   ReportDenovo::append (report_denovo.cpp:59-124), called when d || dm (output.cpp:133-142).  Its idx is set in the for
//   header only: under -out2 without paired_in / paired_out a mate that is not denovo falls through to the write with the idx of
//   the previous iteration, which is 0 (the _fwd file) for both mates.  Reproduced.
__device__ int rpt_file_denovo(const RptArgs& a, uint32_t i, bool d, bool dm) {
  const bool both = d && dm;
  if (a.num_out == 1) return (a.paired_in || d) ? 0 : -1;
  if (a.num_out == 2 && a.out2) {
    if (a.paired_out && !both) return -1;
    return a.paired_in || d ? (int)i : 0;
  }
  if (a.num_out == 2) return both ? 0 : d ? 1 : -1;
  return both ? (int)i : d ? (int)i + 2 : -1;
}

__global__ void rpt_route_kernel(RptArgs a, uint32_t* __restrict__ flags) {
  const bool paired = a.paired_in || a.paired_out || a.mates;
  for (uint32_t r = blockIdx.x * blockDim.x + threadIdx.x; r < a.nreads; r += gridDim.x * blockDim.x) {
    const uint32_t m = paired ? (r ^ 1u) : r;
    const bool empty = a.rec[paired ? (r | 1u) : r].seq_len == 0;   // Readfeed pairs: only the second read is checked (output.cpp:120)
    if (empty) { flags[r] = kRptSkip; continue; }
    const bool h = a.res[r].is_hit;
    uint32_t f = 0;
    int file[3] = {-1, -1, -1};
    if (!paired) {
      file[h ? 0 : 1] = 0;
    } else {
      const bool hm = a.res[m].is_hit;
      file[0] = rpt_file_aligned(a, r & 1u, h, hm);
      file[1] = rpt_file_other(a, r & 1u, h, hm);
    }
    if (a.denovo) {
      const bool d = rpt_is_denovo(a, r);
      if (!paired) { if (d) file[2] = 0; }
      else {
        const bool dm = rpt_is_denovo(a, m);
        if (d || dm) file[2] = rpt_file_denovo(a, r & 1u, d, dm);
      }
    }
    for (uint32_t s = 0; s < 3; ++s)
      if (file[s] >= 0 && (a.fx_mask & (1u << s))) f |= (1u << s) | ((uint32_t)file[s] << (kRptFileShift + 2 * s));
    flags[r] = f;
  }
}

// live alignment slots: key = group (ngroups = not written), value = slot
__global__ void rpt_row_keys_kernel(RptArgs a, const uint32_t* __restrict__ flags, uint32_t* __restrict__ keys, uint32_t* __restrict__ vals) {
  const uint64_t n = a.nslots;
  for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x) {
    const uint32_t r = rpt_read_of(a, i), k = (uint32_t)(i - rpt_slot(a, r, 0));
    uint32_t key = a.ngroups;
    if (k < a.res[r].n_align && !(flags[r] & kRptSkip)) {
      const smr_aln& al = a.aln[i];
      key = rpt_group_of(a, al);
      if (key == a.ngroups) atomicOr(a.err, kRptErrGroup);
      if (al.readlen != a.rec[r].seq_len || al.read_end1 >= (int32_t)a.rec[r].seq_len) atomicOr(a.err, kRptErrLen);
    }
    keys[i] = key; vals[i] = (uint32_t)i;
  }
}

// first[g] = first sorted row of group g (lower bound); first[ngroups] = number of rows
__global__ void rpt_group_first_kernel(const uint32_t* __restrict__ keys, uint64_t n, uint32_t ngroups, uint64_t* __restrict__ first) {
  const uint32_t g = blockIdx.x * blockDim.x + threadIdx.x;
  if (g > ngroups) return;
  uint64_t lo = 0, hi = n;
  while (lo < hi) { const uint64_t mid = (lo + hi) / 2; if (keys[mid] < g) lo = mid + 1; else hi = mid; }
  first[g] = lo;
}

// ---- SAM ----
// QUAL of a row: ReportSam::append reverses read.quality IN PLACE for every minus-strand alignment (report_sam.cpp:125-129), and the
// read object lives for one (index, part) pass: the quality is printed reversed iff an odd number of this read's minus-strand
// alignments of the same (index, part), up to this one, came before in alignv order.
__device__ bool rpt_qual_reversed(const RptArgs& a, uint32_t r, uint32_t k) {
  const smr_aln& al = a.aln[rpt_slot(a, r, k)];
  uint32_t flips = 0;
  for (uint32_t j = 0; j <= k; ++j) {
    const smr_aln& b = a.aln[rpt_slot(a, r, j)];
    flips += b.index_num == al.index_num && b.part == al.part && !b.strand;
  }
  return flips & 1u;
}

__device__ void rpt_sam_prefix(RptSink& o, const RptArgs& a, const RptRec& rc, const smr_aln& al, uint32_t g) {
  rpt_qname(o, a, rc);
  o.s(al.strand ? "\t0\t" : "\t16\t", al.strand ? 3 : 4);
  rpt_ref_name(o, a, a.grp[g], al.ref_num);
  o.c('\t'); o.i((int64_t)al.ref_begin1 + 1);
  o.s("\t255\t", 5);
  rpt_cigar(o, a, al, rc.seq_len);
  o.s("\t*\t0\t0\t", 7);
}
__device__ void rpt_sam_suffix(RptSink& o, const RptArgs& a, const smr_aln& al, const smr_aln_stats& st) {
  o.s("\tAS:i:", 6); o.u(al.score1);
  o.s("\tNM:i:", 6); o.u((uint64_t)st.n_miss + st.n_gap);
  o.c('\n');
}

__global__ void rpt_sam_size_kernel(RptArgs a, const uint32_t* __restrict__ rows, const uint64_t* __restrict__ first, uint64_t* __restrict__ size) {
  const uint64_t n = first[a.ngroups];
  for (uint64_t j = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; j < n; j += (uint64_t)gridDim.x * blockDim.x) {
    const uint32_t i = rows[j], r = rpt_read_of(a, i);
    const smr_aln& al = a.aln[i];
    const RptRec& rc = a.rec[r];
    RptSink o{nullptr, 0};
    rpt_sam_prefix(o, a, rc, al, rpt_group_of(a, al));
    rpt_sam_suffix(o, a, al, a.st[i]);
    size[j] = o.n + rc.seq_len + 1 + (a.fastq ? rc.qual_len : 1);
  }
}

// byte p of a record's sequence (FASTA sequences may span several lines)
struct RptSeqLines {
  const RptArgs& a; const RptRec& rc;
  // calls f(text offset, offset in the sequence, count) for every sequence line, by lane: lanes share the work of each line
  template <class F> __device__ void each(F f) const {
    for (uint32_t l = rc.line + 1; l < (a.fastq ? rc.line + 2 : rc.next); ++l) {
      const uint32_t off = a.spos[l] - a.spos[rc.line], cnt = a.spos[l + 1] - a.spos[l];
      if (cnt) f(rpt_line_beg(a.nl, l), off, cnt);
    }
  }
};

__device__ __forceinline__ char rpt_nt(uint8_t c, bool rc) {   // nt_table (common.hpp:68-77) then ACGTN, complemented for the minus strand
  c &= 0xDF;
  const int v = c == 'A' ? 0 : c == 'C' ? 1 : c == 'G' ? 2 : (c == 'T' || c == 'U') ? 3 : 4;
  return "ACGTN"[rc && v < 4 ? 3 - v : v];
}

__global__ void __launch_bounds__(256) rpt_sam_write_kernel(RptArgs a, const uint32_t* __restrict__ rows, const uint64_t* __restrict__ first,
                                                            const uint64_t* __restrict__ off, char* __restrict__ out) {
  const uint64_t n = first[a.ngroups];
  const unsigned lane = lane_id();
  for (uint64_t j = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; j < n; j += ((uint64_t)gridDim.x * blockDim.x) >> 5) {
    const uint32_t i = rows[j], r = rpt_read_of(a, i);
    const smr_aln al = a.aln[i];
    const RptRec rc = a.rec[r];
    char* dst = out + off[j];
    uint64_t plen = 0;
    if (lane == 0) {
      RptSink o{dst, 0};
      rpt_sam_prefix(o, a, rc, al, rpt_group_of(a, al));
      plen = o.n;
    }
    plen = __shfl_sync(kFull, plen, 0);
    const bool minus = !al.strand;
    const uint32_t L = rc.seq_len;
    char* seq = dst + plen;
    RptSeqLines{a, rc}.each([&](uint64_t src, uint32_t so, uint32_t cnt) {
      for (uint32_t k = lane; k < cnt; k += 32) {
        const uint32_t p = so + k;
        seq[minus ? L - 1 - p : p] = rpt_nt(a.text[src + k], minus);
      }
    });
    char* q = seq + L;
    if (lane == 0) q[0] = '\t';
    ++q;
    uint32_t qlen = 1;
    if (a.fastq) {
      qlen = rc.qual_len;
      const bool rev = rpt_qual_reversed(a, r, (uint32_t)(i - rpt_slot(a, r, 0)));
      for (uint32_t k = lane; k < qlen; k += 32) q[rev ? qlen - 1 - k : k] = (char)a.text[rc.qual + k];
    } else if (lane == 0) {
      q[0] = '*';
    }
    if (lane == 0) {
      RptSink o{q + qlen, 0};
      rpt_sam_suffix(o, a, al, a.st[i]);
    }
  }
}

// ---- BAM (SAMv1 4.2): every SAM row as one BAM record, the same rows in the same order ----
// A record: block_size, refID, pos, l_read_name, mapq, bin, n_cigar_op, flag, l_seq, next_refID, next_pos, tlen (kBamFixed bytes,
// little-endian), read_name with its NUL, the CIGAR words, SEQ (4-bit codes, two per byte), QUAL (phred), the AS and NM tags.
// Records start at any byte, so every field is written byte by byte.
constexpr uint32_t kBamFixed = 36;

__device__ __forceinline__ void bam_le(RptSink& o, uint64_t v, uint32_t n) { for (uint32_t k = 0; k < n; ++k) o.c((char)(v >> (8 * k))); }

// an integer tag (fmt::bam_int_bytes / bam_int_type)
__device__ __forceinline__ void bam_aux_int(RptSink& o, char t0, char t1, uint64_t v) {
  const uint32_t n = fmt::bam_int_bytes(v);
  o.c(t0); o.c(t1); o.c(fmt::bam_int_type(n));
  bam_le(o, v, n);
}

// a read BAM cannot hold: the error bit, and the first such read in *bad
__device__ __forceinline__ void bam_refuse(const RptArgs& a, uint32_t* bad, uint32_t r, uint32_t bit) { atomicOr(a.err, bit); atomicMin(bad, r); }

// the fixed fields, read_name and CIGAR of a row's record; block_size is written, not computed
__device__ void rpt_bam_prefix(RptSink& o, const RptArgs& a, const RptRec& rc, const smr_aln& al, uint32_t g, uint64_t block_size) {
  const RptGroup& G = a.grp[g];
  if (al.ref_num >= G.nref) atomicOr(a.err, kRptErrRef);
  const bool cig_ok = (uint64_t)al.cigar_off + al.cigar_len <= a.cigar_words;
  if (!cig_ok) atomicOr(a.err, kRptErrCigar);
  const uint32_t nc = cig_ok ? al.cigar_len : 0;
  const int64_t lead = rpt_clip_lead(al), trail = rpt_clip_trail(al, rc.seq_len);
  int64_t span = 0;   // reference bases: M and D
  for (uint32_t c = 0; c < nc; ++c) { const uint32_t w = a.cigar[al.cigar_off + c]; if ((w & 0xF) != 1) span += w >> 4; }
  bam_le(o, block_size, 4);
  bam_le(o, G.ref_base + al.ref_num, 4);
  bam_le(o, (uint32_t)al.ref_begin1, 4);
  o.c((char)(rc.name_len + 1)); o.c((char)255);
  bam_le(o, fmt::bam_reg2bin(al.ref_begin1, al.ref_begin1 + span), 2);
  bam_le(o, (lead != 0) + nc + (trail > 0), 2);
  bam_le(o, al.strand ? 0 : 16, 2);
  bam_le(o, rc.seq_len, 4);
  bam_le(o, 0xFFFFFFFFu, 4); bam_le(o, 0xFFFFFFFFu, 4); bam_le(o, 0, 4);
  rpt_qname(o, a, rc); o.c(0);
  if (lead != 0) bam_le(o, (uint64_t)lead << 4 | 4, 4);   // S is op 4; the pool's words are BAM's already (M 0, I 1, D 2)
  for (uint32_t c = 0; c < nc; ++c) bam_le(o, a.cigar[al.cigar_off + c], 4);
  if (trail > 0) bam_le(o, (uint64_t)trail << 4 | 4, 4);
}
__device__ void rpt_bam_suffix(RptSink& o, const smr_aln& al, const smr_aln_stats& st) {
  bam_aux_int(o, 'A', 'S', al.score1);
  bam_aux_int(o, 'N', 'M', (uint64_t)st.n_miss + st.n_gap);
}

// size pass, one thread per row; refuses a QNAME longer than 254 bytes and a FASTQ quality line of another length than the sequence
__global__ void rpt_bam_size_kernel(RptArgs a, const uint32_t* __restrict__ rows, const uint64_t* __restrict__ first, uint64_t* __restrict__ size,
                                    uint32_t* bad) {
  const uint64_t n = first[a.ngroups];
  for (uint64_t j = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; j < n; j += (uint64_t)gridDim.x * blockDim.x) {
    const uint32_t i = rows[j], r = rpt_read_of(a, i);
    const smr_aln& al = a.aln[i];
    const RptRec& rc = a.rec[r];
    if (rc.name_len > 254) bam_refuse(a, bad, r, kRptErrBamName);
    if (a.fastq && rc.qual_len != rc.seq_len) bam_refuse(a, bad, r, kRptErrBamQualLen);
    RptSink o{nullptr, 0};
    rpt_bam_prefix(o, a, rc, al, rpt_group_of(a, al), 0);
    rpt_bam_suffix(o, al, a.st[i]);
    size[j] = o.n + (rc.seq_len + 1) / 2 + rc.seq_len;
  }
}

// write pass, one warp per row.  Lane 0 writes the fixed fields, read_name, CIGAR and tags; the lanes pack SEQ and write QUAL.  SEQ
// goes line by line (RptSeqLines): lane k takes the k-th output byte of the line's positions, and a byte whose other half belongs to
// a line written before is completed with it (the warp syncs between lines).
__global__ void __launch_bounds__(256) rpt_bam_write_kernel(RptArgs a, const uint32_t* __restrict__ rows, const uint64_t* __restrict__ first,
                                                            const uint64_t* __restrict__ off, char* __restrict__ out, uint32_t* bad) {
  const uint64_t n = first[a.ngroups];
  const unsigned lane = lane_id();
  for (uint64_t j = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; j < n; j += ((uint64_t)gridDim.x * blockDim.x) >> 5) {
    const uint32_t i = rows[j], r = rpt_read_of(a, i);
    const smr_aln al = a.aln[i];
    const RptRec rc = a.rec[r];
    char* dst = out + off[j];
    uint64_t plen = 0;
    if (lane == 0) {
      RptSink o{dst, 0};
      rpt_bam_prefix(o, a, rc, al, rpt_group_of(a, al), off[j + 1] - off[j] - 4);
      plen = o.n;
    }
    plen = __shfl_sync(kFull, plen, 0);
    const bool minus = !al.strand;
    const uint32_t L = rc.seq_len;
    uint8_t* seq = (uint8_t*)dst + plen;
    RptSeqLines{a, rc}.each([&](uint64_t src, uint32_t so, uint32_t cnt) {
      const uint32_t p0 = minus ? L - so - cnt : so;   // the line's SEQ positions [p0, p0 + cnt)
      for (uint32_t b = p0 / 2 + lane; b <= (p0 + cnt - 1) / 2; b += 32) {
        uint32_t v = 0;
        bool keep = false;
        for (uint32_t h = 0; h < 2; ++h) {
          const uint32_t p = 2 * b + h;
          if (p >= p0 && p < p0 + cnt) v |= fmt::bam_nt4(rpt_nt(a.text[src + (minus ? L - 1 - p : p) - so], minus)) << (h ? 0 : 4);
          else if (p < L) keep = true;   // lines come in text order: the other half was written unless it comes later
        }
        if (keep && (minus ? 2 * b + 1 >= p0 + cnt : 2 * b < p0)) v |= seq[b];
        seq[b] = (uint8_t)v;
      }
      __syncwarp();
    });
    uint8_t* q = seq + (L + 1) / 2;
    if (a.fastq) {   // the size pass refused a quality line of another length than L
      const bool rev = rpt_qual_reversed(a, r, (uint32_t)(i - rpt_slot(a, r, 0)));
      for (uint32_t k = lane; k < L; k += 32) {
        const uint8_t c = a.text[rc.qual + k];
        if (c < '!' || c > '~') bam_refuse(a, bad, r, kRptErrBamQualByte);
        q[rev ? L - 1 - k : k] = (uint8_t)(c - 33);
      }
    } else {
      for (uint32_t k = lane; k < L; k += 32) q[k] = 0xFF;
    }
    if (lane == 0) {
      RptSink o{(char*)q + L, 0};
      rpt_bam_suffix(o, al, a.st[i]);
    }
  }
}

// ---- tabular BLAST (one thread per row) ----
__device__ void rpt_blast_row(RptSink& o, const RptArgs& a, const RptRec& rc, const smr_aln& al, const smr_aln_stats& st, uint32_t g) {
  const RptGroup& G = a.grp[g];
  rpt_qname(o, a, rc); o.c('\t');
  rpt_ref_name(o, a, G, al.ref_num); o.c('\t');
  o.g3((double)st.n_match / (double)(st.n_miss + st.n_gap + st.n_match) * 100); o.c('\t');
  o.i((int64_t)al.read_end1 - al.read_begin1 + 1); o.c('\t');
  o.u(st.n_miss); o.c('\t');
  o.u(st.n_gap); o.c('\t');
  o.i((int64_t)al.read_begin1 + 1); o.c('\t');
  o.i((int64_t)al.read_end1 + 1); o.c('\t');
  o.i((int64_t)al.ref_begin1 + 1); o.c('\t');
  o.i((int64_t)al.ref_end1 + 1); o.c('\t');
  o.g3(G.evalue[al.score1]); o.c('\t');
  o.u(G.bits[al.score1]);
  for (uint32_t c = 0; c < a.ncols; ++c) {
    o.c('\t');
    if (a.cols[c] == kColCigar) {
      rpt_cigar(o, a, al, rc.seq_len);
    } else if (a.cols[c] == kColQcov) {
      const int32_t span = al.read_end1 - al.read_begin1 + 1;
      o.g3((double)(span < 0 ? -span : span) / (double)al.readlen * 100);
    } else {
      o.c(al.strand ? '+' : '-');
    }
  }
  o.c('\n');
}

__global__ void rpt_blast_kernel(RptArgs a, const uint32_t* __restrict__ rows, const uint64_t* __restrict__ first, uint64_t* __restrict__ size,
                                 const uint64_t* __restrict__ off, char* __restrict__ out) {
  const uint64_t n = first[a.ngroups];
  for (uint64_t j = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; j < n; j += (uint64_t)gridDim.x * blockDim.x) {
    const uint32_t i = rows[j];
    const smr_aln& al = a.aln[i];
    RptSink o{out ? out + off[j] : nullptr, 0};
    rpt_blast_row(o, a, a.rec[rpt_read_of(a, i)], al, a.st[i], rpt_group_of(a, al));
    if (size) size[j] = o.n;
  }
}

// ---- pairwise BLAST (-blast 0): report_blast.cpp:136-251 ----
// Per row: the header (Sequence ID / Query ID / Score, bits, Expect, strand, blank line), then the CIGAR's columns in blocks of 60:
//   "Target: " q0+1 (width 8) "    " <ref chars, '-' for I>  "    " q1 "\n"
//   20 spaces                         <'|' equal, '*' differ, ' ' for I and D>
//   "\nQuery: " p0+1 (width 9) "    " <read chars, '-' for D> "    " p1 "\n\n"
// q0 / p0: the 0-based reference / read positions at the block's first column; q1 / p1: the positions after its last.  The reference's
// three passes with their goto / left / e carry-over come down to this plain chunking of the columns.
constexpr uint32_t kPwCols = 60;

__device__ __forceinline__ uint32_t rpt_digits(uint64_t v) { uint32_t d = 1; while (v >= 10) { v /= 10; ++d; } return d; }

// byte layout of one block of n columns, relative to its start
struct RptPwBlock {
  uint32_t ref, mid, qry, bytes;   // offsets of the three column runs; size of the block
  __device__ RptPwBlock(uint32_t q0, uint32_t p0, uint32_t n, uint32_t q1, uint32_t p1) {
    const uint32_t wt = max(8u, rpt_digits((uint64_t)q0 + 1)), wq = max(9u, rpt_digits((uint64_t)p0 + 1));
    ref = 8 + wt + 4;
    mid = ref + n + 4 + rpt_digits(q1) + 1 + 20;
    qry = mid + n + 8 + wq + 4;
    bytes = qry + n + 4 + rpt_digits(p1) + 2;
  }
};

__device__ void rpt_pw_header(RptSink& o, const RptArgs& a, const RptRec& rc, const smr_aln& al, const RptGroup& G) {
  o.s("Sequence ID: ", 13); rpt_ref_name(o, a, G, al.ref_num); o.c('\n');
  o.s("Query ID: ", 10); rpt_qname(o, a, rc); o.c('\n');
  o.s("Score: ", 7); o.u(al.score1); o.s(" bits (", 7); o.u(G.bits[al.score1]);
  o.s(")\tExpect: ", 10); o.g3(G.evalue[al.score1]);
  o.s("\tstrand: ", 9); o.c(al.strand ? '+' : '-'); o.s("\n\n", 2);
}

// v right-aligned in a field of w (ss.width(w); a longer number is not cut)
__device__ void rpt_pw_num(RptSink& o, uint64_t v, uint32_t w) {
  for (uint32_t d = rpt_digits(v); d < w; ++d) o.c(' ');
  o.u(v);
}

// size pass, one thread per row: walks the CIGAR ops, not the columns.  A column past the read or the reference is kRptErrSpan.
__global__ void rpt_pw_size_kernel(RptArgs a, const uint32_t* __restrict__ rows, const uint64_t* __restrict__ first, uint64_t* __restrict__ size) {
  const uint64_t n = first[a.ngroups];
  for (uint64_t j = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; j < n; j += (uint64_t)gridDim.x * blockDim.x) {
    const uint32_t i = rows[j];
    const smr_aln& al = a.aln[i];
    const RptRec& rc = a.rec[rpt_read_of(a, i)];
    const RptGroup& G = a.grp[rpt_group_of(a, al)];
    RptSink o{nullptr, 0};
    rpt_pw_header(o, a, rc, al, G);
    size[j] = o.n;
    if (al.ref_num >= G.nref) continue;   // kRptErrRef is set
    if ((uint64_t)al.cigar_off + al.cigar_len > a.cigar_words) { atomicOr(a.err, kRptErrCigar); continue; }
    if (al.ref_begin1 < 0 || al.read_begin1 < 0) { atomicOr(a.err, kRptErrSpan); continue; }
    uint32_t q = (uint32_t)al.ref_begin1, p = (uint32_t)al.read_begin1, q0 = q, p0 = p, fill = 0;
    uint64_t bytes = o.n;
    for (uint32_t c = 0; c < al.cigar_len; ++c) {
      const uint32_t w = a.cigar[al.cigar_off + c], op = w & 0xF;
      for (uint32_t len = w >> 4; len;) {
        const uint32_t take = min(len, kPwCols - fill);
        if (op != 1) q += take;
        if (op <= 1) p += take;
        fill += take; len -= take;
        if (fill == kPwCols) { bytes += RptPwBlock(q0, p0, fill, q, p).bytes; fill = 0; q0 = q; p0 = p; }
      }
    }
    if (fill) bytes += RptPwBlock(q0, p0, fill, q, p).bytes;
    if (q > G.ref_off[al.ref_num + 1] - G.ref_off[al.ref_num] || p > rc.seq_len) atomicOr(a.err, kRptErrSpan);
    size[j] = bytes;
  }
}

// read char at position p of the read as aligned (reverse-complemented on the minus strand), as SAM's SEQ prints it
__device__ __forceinline__ char rpt_read_char(const RptArgs& a, const RptRec& rc, uint32_t p, bool minus) {
  const uint32_t pos = minus ? rc.seq_len - 1 - p : p, base = a.spos[rc.line];
  uint32_t l = rc.line + 1;
  if (!a.fastq && rc.next > rc.line + 2) {   // FASTA over several lines: the last line that starts at or before pos
    uint32_t hi = rc.next - 1;
    while (l < hi) { const uint32_t m = (l + hi + 1) / 2; if (a.spos[m] - base <= pos) l = m; else hi = m - 1; }
  }
  return rpt_nt(a.text[rpt_line_beg(a.nl, l) + pos - (a.spos[l] - base)], minus);
}

// write pass, one warp per row.  Lane 0 writes the header and the numbers of each block; the warp walks the CIGAR one block at a
// time, carrying the block's starting (op, offset in op, q, p), and lanes k and k + 32 take the block's columns k and k + 32.
__global__ void __launch_bounds__(256) rpt_pw_write_kernel(RptArgs a, const uint32_t* __restrict__ rows, const uint64_t* __restrict__ first,
                                                           const uint64_t* __restrict__ off, char* __restrict__ out) {
  const uint64_t n = first[a.ngroups];
  const unsigned lane = lane_id();
  for (uint64_t j = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; j < n; j += ((uint64_t)gridDim.x * blockDim.x) >> 5) {
    const uint32_t i = rows[j];
    const smr_aln& al = a.aln[i];
    const RptRec& rc = a.rec[rpt_read_of(a, i)];
    const RptGroup& G = a.grp[rpt_group_of(a, al)];
    char* dst = out + off[j];
    uint64_t at = 0;
    if (lane == 0) {
      RptSink o{dst, 0};
      rpt_pw_header(o, a, rc, al, G);
      at = o.n;
    }
    at = __shfl_sync(kFull, at, 0);
    const uint8_t* ref = G.refseq + G.ref_off[al.ref_num];
    const uint32_t* cig = a.cigar + al.cigar_off;
    const bool minus = !al.strand;
    uint32_t c = 0, used = 0, q = (uint32_t)al.ref_begin1, p = (uint32_t)al.read_begin1;
    while (c < al.cigar_len) {
      const uint32_t q0 = q, p0 = p;
      uint32_t fill = 0;
      char r0 = 0, m0 = 0, s0 = 0, r1 = 0, m1 = 0, s1 = 0;   // this lane's columns lane and lane + 32
      while (fill < kPwCols && c < al.cigar_len) {
        const uint32_t w = cig[c], op = w & 0xF, take = min((w >> 4) - used, kPwCols - fill);
        auto col = [&](uint32_t k, char& r, char& m, char& s) {
          if (k < fill || k >= fill + take) return;
          const uint32_t d = k - fill;
          r = op == 1 ? '-' : "ACGTN"[min((uint32_t)ref[q + d], 4u)];
          s = op > 1 ? '-' : rpt_read_char(a, rc, p + d, minus);
          m = op == 0 ? (r == s ? '|' : '*') : ' ';
        };
        col(lane, r0, m0, s0);
        col(lane + 32, r1, m1, s1);
        if (op != 1) q += take;
        if (op <= 1) p += take;
        fill += take; used += take;
        if (used == w >> 4) { ++c; used = 0; }
      }
      if (!fill) break;   // only empty ops were left
      const RptPwBlock b(q0, p0, fill, q, p);
      char* blk = dst + at;
      if (lane < fill) { blk[b.ref + lane] = r0; blk[b.mid + lane] = m0; blk[b.qry + lane] = s0; }
      if (lane + 32 < fill) { blk[b.ref + lane + 32] = r1; blk[b.mid + lane + 32] = m1; blk[b.qry + lane + 32] = s1; }
      if (lane == 0) {
        RptSink o{blk, 0};
        o.s("Target: ", 8); rpt_pw_num(o, (uint64_t)q0 + 1, 8); o.s("    ", 4);
        o.n = b.ref + fill; o.s("    ", 4); o.u(q); o.c('\n'); o.s("                    ", 20);
        o.n = b.mid + fill; o.s("\nQuery: ", 8); rpt_pw_num(o, (uint64_t)p0 + 1, 9); o.s("    ", 4);
        o.n = b.qry + fill; o.s("    ", 4); o.u(p); o.s("\n\n", 2);
      }
      at += b.bytes;
    }
  }
}

// ---- aligned / other / aligned_denovo reads: write_a_read (report_fx_base.cpp:176-181) ----
// the stream of kind s of a read with route flags f: the kinds one after another, num_out files each, in the reference's file order
__device__ __forceinline__ uint32_t rpt_fx_stream(const RptArgs& a, uint32_t f, uint32_t s) { return s * a.num_out + ((f >> (kRptFileShift + 2 * s)) & 3u); }

__global__ void rpt_fx_size_kernel(RptArgs a, const uint32_t* __restrict__ flags, uint64_t* __restrict__ size, uint64_t stride) {
  for (uint32_t r = blockIdx.x * blockDim.x + threadIdx.x; r < a.nreads; r += gridDim.x * blockDim.x) {
    const RptRec& rc = a.rec[r];
    const uint64_t len = (uint64_t)rc.hdr_len + rc.seq_len + 2 + (a.fastq ? rc.qual_len + 3 : 0);
    const uint32_t f = flags[r];
    for (uint32_t s = 0; s < 3; ++s)   // route masked the files not asked for; the sizes are zeroed before
      if (f & (1u << s)) size[rpt_fx_stream(a, f, s) * stride + r] = len;
  }
}

__device__ __forceinline__ void rpt_warp_copy(char* dst, const uint8_t* src, uint64_t n, unsigned lane) {
  for (uint64_t k = lane; k < n; k += 32) dst[k] = (char)src[k];
}

// off: one exclusive scan over the sizes of the read files (stride nreads + 1), so off already includes the files before; *base = start
// of the first read file in the output
__global__ void __launch_bounds__(256) rpt_fx_write_kernel(RptArgs a, const uint32_t* __restrict__ flags, const uint64_t* __restrict__ off,
                                                           uint64_t stride, const uint64_t* __restrict__ base, char* __restrict__ out) {
  const unsigned lane = lane_id();
  for (uint32_t r = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; r < a.nreads; r += (gridDim.x * blockDim.x) >> 5) {
    const uint32_t f = flags[r];
    const RptRec rc = a.rec[r];
    for (uint32_t s = 0; s < 3; ++s) {
      if (!(f & (1u << s))) continue;
      char* dst = out + base[0] + off[rpt_fx_stream(a, f, s) * stride + r];
      if (rc.verbatim) { rpt_warp_copy(dst, a.text + rc.hdr, (uint64_t)rc.hdr_len + rc.seq_len + rc.qual_len + 5, lane); continue; }
      rpt_warp_copy(dst, a.text + rc.hdr, rc.hdr_len, lane);
      char* seq = dst + rc.hdr_len + 1;
      RptSeqLines{a, rc}.each([&](uint64_t src, uint32_t so, uint32_t cnt) { rpt_warp_copy(seq + so, a.text + src, cnt, lane); });
      char* q = seq + rc.seq_len;
      if (lane == 0) { dst[rc.hdr_len] = '\n'; q[0] = '\n'; if (a.fastq) { q[1] = '+'; q[2] = '\n'; q[3 + rc.qual_len] = '\n'; } }
      if (a.fastq) rpt_warp_copy(q + 3, a.text + rc.qual, rc.qual_len, lane);
    }
  }
}

// stream offsets: SAM groups, BLAST groups, the nfx read files (aligned, other, denovo; num_out files each): 2 * ngroups + nfx + 1 entries
__global__ void rpt_stream_off_kernel(const uint64_t* __restrict__ first, uint32_t ngroups, const uint64_t* __restrict__ sam_off,
                                      const uint64_t* __restrict__ blast_off, const uint64_t* __restrict__ fx_off, uint32_t nreads, uint64_t stride,
                                      uint32_t nfx, uint64_t* __restrict__ so) {
  if (threadIdx.x != 0 || blockIdx.x != 0) return;
  const uint64_t sam_total = sam_off[first[ngroups]];
  for (uint32_t g = 0; g <= ngroups; ++g) so[g] = sam_off[first[g]];
  for (uint32_t g = 0; g <= ngroups; ++g) so[ngroups + g] = sam_total + blast_off[first[g]];
  for (uint32_t s = 0; s < nfx; ++s) so[2 * ngroups + 1 + s] = so[2 * ngroups] + fx_off[s * stride + nreads];   // fx_off: one scan over them all
}

}  // namespace smr
