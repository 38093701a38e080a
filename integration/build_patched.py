#!/usr/bin/env python
"""integration/build_patched.py -- compiles the shim FOR REAL (SURVEY 8b, VERDICT row g1): makes patched COPIES of three reference translation
units under oracle/_ref/build/patched/ (git-ignored scratch; the reference tree is read-only and stays untouched, nothing of it enters this
repository), each edit a call-site substitution, compiles them with the oracle build's flags and links

    oracle/_ref/bin/starling2_sx   germline caller: computeSampleDiploidSiteGenotype -> sx_site_gl_germline (K2a), haplotype alignment -> sx_global_align (K3),
                                   getVariantAlleleGroupGenotypeLhoodsForSample -> sx_indel_gl (K5), process_pos_snp_continuous -> sx_site_continuous (K2c),
                                   the continuous indel GQ -> sx_cont_qscore
    oracle/_ref/bin/strelka2_sx    somatic caller:  position_somatic_snv_call -> sx_site_gl_somatic (K2b), get_somatic_indel -> sx_somatic_indel (K5b)
    oracle/_ref/bin/starling2, strelka2   the unmodified reference binaries (oracle/build_ref.sh --bins)

against strelka_b200/csrc/libstrelka_b200.so.  It also stages the bundled demo inputs (BAMs, reference, model files, expected VCFs) under
oracle/_ref/demo/ so that the GPU box -- which has no /root/reference -- can run tests/test_zzzzz_gpu_demo_vcf.py.  Run here (needs the reference)."""
import os
import re
import shutil
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = os.environ.get("STRELKA_REFERENCE", "/root/reference")
B = os.path.join(ROOT, "oracle", "_ref", "build")
OUT = os.path.join(ROOT, "oracle", "_ref", "bin")
DEMO = os.path.join(ROOT, "oracle", "_ref", "demo")
L = os.path.join(REF, "src", "c++", "lib")

# the K2c route at the top of process_pos_snp_continuous, and the continuous indel GQ through sx_cont_qscore
CONTINUOUS_SITE = r'''starling_pos_processor::
process_pos_snp_continuous(const pos_t pos)
{
    if (sx_shim::enabled() && getSampleCount() <= SX_CONT_MAX_SAMPLES)
    {
        // K2c's records, turned into loci by the reference's own updateSiteSampleInfo / updateContinuousSiteSampleInfo / add_site
        const unsigned sxS(getSampleCount());
        std::vector<const snp_pos_info*> sxRaw;
        for (unsigned s(0); s < sxS; ++s) sxRaw.push_back(&sample(s).cleanedPileup.rawPileup());
        sx_shim::ContinuousSite sxSite;
        sx_shim::continuous_site(_opt, sxRaw, _ref.get_base(pos), is_forced_output_pos(pos), pos, sxSite);
        const uint8_t sxRefBase(base_to_id(_ref.get_base(pos)));
        for (unsigned r(0); r < sxSite.loci.size(); ++r)
        {
            const sx_cont_locus& L(sxSite.loci[r]);
            const bool isRefAllele(L.alt == SX_CONT_REF_LOCUS);
            std::unique_ptr<GermlineContinuousSiteLocusInfo> locusPtr(new GermlineContinuousSiteLocusInfo(sxS, pos, sxRefBase, L.forced != 0));
            if (not isRefAllele) locusPtr->addAltSiteAllele(static_cast<BASE_ID::index_t>(L.alt));
            int qual(0);
            for (unsigned s(0); s < sxS; ++s)
            {
                const sx_cont_sample& E(sxSite.samples[r * sxS + s]);
                const CleanedPileup& cpi(sample(s).cleanedPileup);
                auto& sampleInfo(locusPtr->getSample(s));
                sampleInfo.supportCounts.setAltCount(isRefAllele ? 0 : 1);
                auto& fwd(sampleInfo.supportCounts.getCounts(true));
                auto& rev(sampleInfo.supportCounts.getCounts(false));
                if (E.ref_fwd) fwd.incrementAlleleCount(0, E.ref_fwd);
                if (E.ref_rev) rev.incrementAlleleCount(0, E.ref_rev);
                if (E.alt_fwd) fwd.incrementAlleleCount(1, E.alt_fwd);
                if (E.alt_rev) rev.incrementAlleleCount(1, E.alt_rev);
                fwd.nonConfidentCount += E.non_confident_fwd;
                rev.nonConfidentCount += E.non_confident_rev;
                double sb(E.strand_bias);
                if ((not isRefAllele) && sx_shim::near_strand_bias_boundary(sb)) sb = sx_shim::reference_sample_strand_bias(cpi.cleanedPileup(), L.alt);
                updateSiteSampleInfo(_opt, s, cpi, false, sb, *locusPtr);
                updateContinuousSiteSampleInfo(s, isRefAllele ? 0 : 1, *locusPtr);
                sampleInfo.maxGenotypeIndexPolymorphic = (E.gt == SX_CONT_GT_HOM) ? VcfGenotype(1, 1) : (E.gt == SX_CONT_GT_HET) ? VcfGenotype(0, 1) : VcfGenotype(0, 0);
                const int gq((E.status & SX_CONT_ST_QSCORE_TIE) ? starling_continuous_variant_caller::getAlleleSequencingErrorQscore(
                                 E.allele_depth, E.total_depth, _opt.continuousFrequencyCallerExpectedObservationQuality, _opt.continuousFrequencyCallerMaxQscore)
                             : E.gq);
                sampleInfo.gqx = sampleInfo.genotypeQualityPolymorphic = gq;
                qual = std::max(qual, gq);
            }
            locusPtr->hpol = get_snp_hpol_size(pos, _ref);
            locusPtr->anyVariantAlleleQuality = 0;
            if (not isRefAllele)
            {
                double sb(L.strand_bias);
                if (sx_shim::near_strand_bias_boundary(sb)) sb = starling_continuous_variant_caller::strandBias(L.sb_fwd_alt, L.sb_rev_alt, L.sb_fwd_other, L.sb_rev_other);
                locusPtr->getSiteAlleles()[0].strandBias = sb;
                locusPtr->anyVariantAlleleQuality = qual;
            }
            _gvcfer->add_site(std::move(locusPtr));
        }
        return;
    }
'''
CONTINUOUS_INDEL_GQ = r'''sampleInfo.gqx = sampleInfo.genotypeQualityPolymorphic =
                         (sx_shim::enabled() ? sx_shim::cont_qscore(opt, indelSampleInfo.legacyReportInfo.n_confident_indel_reads,
                                                                     indelSampleInfo.legacyReportInfo.total_confident_reads())
                          : starling_continuous_variant_caller::getAlleleSequencingErrorQscore(
                             indelSampleInfo.legacyReportInfo.n_confident_indel_reads,
                             indelSampleInfo.legacyReportInfo.total_confident_reads(),
                             opt.continuousFrequencyCallerExpectedObservationQuality,
                             opt.continuousFrequencyCallerMaxQscore));'''

# (file, [(regex of the call site, replacement)], extra text put after the file's last #include, extra defines)
EDITS = [
    ("applications/starling/starling_pos_processor.cpp",
     [(r"dopt\.pdcaller\(\)\.position_snp_call_pprob_digt\(\s*opt,\s*good_epi,\s*dgt,\s*opt\.is_all_sites\(\)\);",
       "if (sx_shim::enabled()) sx_shim::site_gl_germline(opt, sif.cleanedPileup.rawPileup(), opt.is_all_sites(), dgt);\n"
       "    else dopt.pdcaller().position_snp_call_pprob_digt(opt, good_epi, dgt, opt.is_all_sites());"),
      (r"getVariantAlleleGroupGenotypeLhoodsForSample\(\s*opt,\s*dopt,\s*sample_opt,\s*callerPloidy,\s*sampleIndex,\s*alleleGroup,\s*contrastGroup,\s*"
       r"genotypeLogLhood,\s*sampleInfo\.supportCounts\);",
       "if (sx_shim::enabled()) sx_shim::germline_indel(opt, dopt, sample_opt, callerPloidy, sampleIndex, alleleGroup, contrastGroup, genotypeLogLhood,\n"
       "                                                sampleInfo.supportCounts);\n"
       "    else getVariantAlleleGroupGenotypeLhoodsForSample(opt, dopt, sample_opt, callerPloidy, sampleIndex, alleleGroup, contrastGroup,\n"
       "                                                      genotypeLogLhood, sampleInfo.supportCounts);"),
      # process_pos_snp_continuous (:926-996): K2c first; more samples than SX_CONT_MAX_SAMPLES keep the reference code below
      (r"starling_pos_processor::\s*process_pos_snp_continuous\(const pos_t pos\)\s*\{", CONTINUOUS_SITE),
      # the continuous indel genotype's GQ (:2026-2030) through sx_cont_qscore
      (r"sampleInfo\.gqx = sampleInfo\.genotypeQualityPolymorphic =\s*starling_continuous_variant_caller::getAlleleSequencingErrorQscore\(\s*"
       r"indelSampleInfo\.legacyReportInfo\.n_confident_indel_reads,\s*indelSampleInfo\.legacyReportInfo\.total_confident_reads\(\),\s*"
       r"opt\.continuousFrequencyCallerExpectedObservationQuality,\s*opt\.continuousFrequencyCallerMaxQscore\);", CONTINUOUS_INDEL_GQ)],
     "#define SX_SHIM_GERMLINE\n#define SX_SHIM_CONTINUOUS\n"),
    ("starling_common/ActiveRegionProcessor.cpp",
     [(r"_aligner\.align\(haplotypeSeq\.cbegin\(\),\s*haplotypeSeq\.cend\(\),\s*_refSegment\.cbegin\(\),\s*_refSegment\.cend\(\),\s*result\);",
       "if (sx_shim::enabled()) sx_shim::global_align(_aligner.getScores(), haplotypeSeq, _refSegment, result);\n"
       "    else _aligner.align(haplotypeSeq.cbegin(),haplotypeSeq.cend(),_refSegment.cbegin(),_refSegment.cend(),result);")], ""),
    ("applications/strelka/strelka_pos_processor.cpp",
     [(r"_dopt\.sscaller_strand_grid\(\)\.position_somatic_snv_call\(\s*normal_cpi_ptr\[0\]->getExtendedPosInfo\(\),\s*tumor_cpi_ptr\[0\]->getExtendedPosInfo\(\),\s*"
       r"normal_epi_t2_ptr,\s*tumor_epi_t2_ptr,\s*isComputeNonSomatic,\s*sgtg\);",
       "if (sx_shim::enabled()) sx_shim::site_gl_somatic(_opt, normal_cpi_ptr[0]->rawPileup(), tumor_cpi_ptr[0]->rawPileup(), isComputeNonSomatic, sgtg);\n"
       "        else _dopt.sscaller_strand_grid().position_somatic_snv_call(normal_cpi_ptr[0]->getExtendedPosInfo(), tumor_cpi_ptr[0]->getExtendedPosInfo(),\n"
       "                                                                    normal_epi_t2_ptr, tumor_epi_t2_ptr, isComputeNonSomatic, sgtg);"),
      (r"_dopt\.sicaller_grid\(\)\.get_somatic_indel\(\s*_opt,\s*_dopt,\s*normal_sif\.sampleOptions,\s*tumor_sif\.sampleOptions,\s*indelKey,\s*indelData,\s*NORMAL,\s*TUMOR,\s*"
       r"is_use_alt_indel,\s*siInfo\.sindel\);",
       "if (sx_shim::enabled() && is_use_alt_indel) sx_shim::somatic_indel(_opt, _dopt, normal_sif.sampleOptions, tumor_sif.sampleOptions, indelKey, indelData, NORMAL, TUMOR,\n"
       "                                                                 siInfo.sindel);\n"
       "            else _dopt.sicaller_grid().get_somatic_indel(_opt, _dopt, normal_sif.sampleOptions, tumor_sif.sampleOptions, indelKey, indelData, NORMAL, TUMOR,\n"
       "                                                         is_use_alt_indel, siInfo.sindel);")], "#define SX_SHIM_SOMATIC\n"),
]


def sh(cmd, **kw):
    subprocess.check_call(cmd, **kw)


def main():
    if not os.path.isdir(L):
        print("build_patched.py: reference tree not found; nothing to do", file=sys.stderr)
        return 0
    sh([os.path.join(ROOT, "oracle", "build_ref.sh"), "--bins"])
    os.makedirs(OUT, exist_ok=True)
    pdir = os.path.join(B, "patched")
    os.makedirs(pdir, exist_ok=True)
    inc = [f"-I{B}/gen", f"-I{L}", f"-I{B}/boost_1_58_0_subset", f"-I{B}/htslib-1.7-6-g6d2bfb7", f"-I{B}/rapidjson-1.1.0/include", f"-I{B}/CodeMin-1.0.5/include",
           f"-I{ROOT}/include", f"-I{ROOT}/strelka_b200/host", f"-I{ROOT}/integration"]
    flags = ["-std=c++11", "-O3", "-fomit-frame-pointer", "-fPIC", "-w"]
    objs = {}
    for rel, subs, pre in EDITS:
        src = open(os.path.join(L, rel)).read()
        for pat, rep in subs:
            src, n = re.subn(pat, lambda m, rep=rep: rep, src, count=1, flags=re.S)
            assert n == 1, f"call site not found in {rel}: {pat[:60]}"
        # the shim header goes after the file's last #include (its own includes need the reference's include paths only)
        last = [m for m in re.finditer(r"^#include[^\n]*\n", src, flags=re.M)][-1]
        src = src[: last.end()] + pre + '#include "sx_shim.hh"\n' + src[last.end():]
        dst = os.path.join(pdir, rel.replace("/", "_"))
        open(dst, "w").write(src)
        obj = dst[:-4] + ".o"
        sh(["g++"] + flags + inc + [f"-I{os.path.dirname(os.path.join(L, rel))}", "-c", dst, "-o", obj])
        objs[rel] = obj
    lib = os.path.join(ROOT, "strelka_b200", "csrc")
    tail = [os.path.join(B, "libboost.a"), os.path.join(B, "htslib-1.7-6-g6d2bfb7", "libhts.a"), "-lz", "-lpthread", f"-L{lib}", "-lstrelka_b200", f"-Wl,-rpath,{lib}",
            "-Wl,-rpath,$ORIGIN/../../../strelka_b200/csrc"]
    # the patched objects come first on the link line: the archive members of the same translation units are then not pulled
    sh(["g++", "-o", os.path.join(OUT, "starling2_sx"), os.path.join(B, "obj", "main_starling2.o"), objs["applications/starling/starling_pos_processor.cpp"],
        objs["starling_common/ActiveRegionProcessor.cpp"], "-Wl,--start-group", os.path.join(B, "libapp_starling.a"), os.path.join(B, "libcommon.a"), "-Wl,--end-group"] + tail)
    sh(["g++", "-o", os.path.join(OUT, "strelka2_sx"), os.path.join(B, "obj", "main_strelka2.o"), objs["applications/strelka/strelka_pos_processor.cpp"],
        "-Wl,--start-group", os.path.join(B, "libapp_strelka.a"), os.path.join(B, "libcommon.a"), "-Wl,--end-group"] + tail)
    for b in ("starling2", "strelka2"):
        shutil.copy2(os.path.join(ROOT, "oracle", "_ref", b), os.path.join(OUT, b))
    # demo inputs for the GPU box
    os.makedirs(os.path.join(DEMO, "data"), exist_ok=True)
    os.makedirs(os.path.join(DEMO, "expected"), exist_ok=True)
    os.makedirs(os.path.join(DEMO, "config"), exist_ok=True)
    for f in os.listdir(os.path.join(REF, "src", "demo", "data")):
        if not f.endswith(".txt"):
            shutil.copy2(os.path.join(REF, "src", "demo", "data", f), os.path.join(DEMO, "data", f))
    for f in os.listdir(os.path.join(REF, "src", "demo", "expectedResults")):
        shutil.copy2(os.path.join(REF, "src", "demo", "expectedResults", f), os.path.join(DEMO, "expected", f))
    # the mitochondrial demo (src/demo/runMitoWorkflowDemo.bash): chrM, called with --call-continuous-vf
    os.makedirs(os.path.join(DEMO, "dataMito"), exist_ok=True)
    for f in os.listdir(os.path.join(REF, "src", "demo", "dataMito")):
        shutil.copy2(os.path.join(REF, "src", "demo", "dataMito", f), os.path.join(DEMO, "dataMito", f))
    shutil.copy2(os.path.join(REF, "src", "demo", "expectedResultsMito", "genome.vcf.gz"), os.path.join(DEMO, "expected", "mito.genome.vcf.gz"))
    cfg = os.path.join(REF, "src", "config")
    for f in ("empiricalVariantScoring/models/germlineSNVScoringModels.json", "empiricalVariantScoring/models/germlineIndelScoringModels.json",
              "empiricalVariantScoring/models/somaticSNVScoringModels.json", "empiricalVariantScoring/models/somaticIndelScoringModels.json",
              "indelErrorModel/models/indelErrorModel.json", "indelErrorModel/models/theta.json"):
        shutil.copy2(os.path.join(cfg, f), os.path.join(DEMO, "config", os.path.basename(f)))
    print("built", OUT, "and staged", DEMO)
    return 0


if __name__ == "__main__":
    sys.exit(main())
