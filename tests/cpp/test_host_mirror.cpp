// test_host_mirror.cpp -- the C++ host mirror (strelka_b200/host/strelka_b200.hh) on the GPU, written the way the reference's own
// unit tests read (alignment/test/GlobalAlignerTest.cpp, starling_common/test/starling_read_align_test.cpp):
//   * GlobalAligner<int>::align on the reference's 22 known-answer cases (CIGAR, beginPos, score)
//   * ReadAlignBatch::scoreCandidateAlignments on reference-shaped CandidateAlignments, compared bit-for-bit with the reference's
//     scoreCandidateAlignment results frozen in tests/golden/k1_cases.tsv
// Build/run: see tests/test_gpu_parity.py::test_cpp_host_mirror.
#include "strelka_b200.hh"

#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <fstream>
#include <iostream>
#include <map>
#include <sstream>

static std::vector<std::string> split(const std::string& s, char d)
{
    std::vector<std::string> out;
    std::string cur;
    std::istringstream is(s);
    while (std::getline(is, cur, d)) out.push_back(cur);
    return out;
}

int main(int argc, char** argv)
{
    if (argc < 2)
    {
        std::cerr << "usage: test_host_mirror <tests/golden dir>\n";
        return 2;
    }
    const std::string dir(argv[1]);
    int failures(0), checks(0);
    try
    {
        sx::Context ctx(0);
        // ---- GlobalAligner goldens
        {
            std::ifstream in(dir + "/global_aligner_goldens.tsv");
            std::string line;
            while (std::getline(in, line))
            {
                const std::vector<std::string> f(split(line, '\t'));
                if (f.size() < 14) continue;
                const sx::AlignmentScores<int> scores(atoi(f[3].c_str()), atoi(f[4].c_str()), atoi(f[5].c_str()), atoi(f[6].c_str()), atoi(f[7].c_str()),
                                                      atoi(f[8].c_str()), atoi(f[9].c_str()) != 0, atoi(f[10].c_str()) != 0);
                const sx::GlobalAligner<int> aligner(ctx, scores);
                sx::AlignmentResult<int> result;
                const std::string &seq(f[1]), &ref(f[2]);
                aligner.align(seq.begin(), seq.end(), ref.begin(), ref.end(), result);
                ++checks;
                if (sx::apath_to_cigar(result.align.apath) != f[11] || result.align.beginPos != atoi(f[12].c_str()) ||
                    (f[13] != "NA" && result.score != atoi(f[13].c_str())))
                {
                    ++failures;
                    std::cerr << "FAIL " << f[0] << ": got " << sx::apath_to_cigar(result.align.apath) << " @" << result.align.beginPos << " score " << result.score
                              << ", want " << f[11] << " @" << f[12] << " score " << f[13] << "\n";
                }
            }
        }
        // ---- scoreCandidateAlignment cases
        {
            std::ifstream in(dir + "/k1_cases.tsv");
            std::string line;
            sx::ReadAlignBatch batch;
            std::vector<uint64_t> want;
            unsigned regionReadBase(0), nReads(0);
            // candidacy is a property of the key within a region's IndelBuffer
            while (std::getline(in, line))
            {
                const std::vector<std::string> f(split(line, '\t'));
                if (f[0] == "REGION")
                {
                    batch.beginRegion(f[1], atoi(f[2].c_str()));
                    regionReadBase = nReads;
                }
                else if (f[0] == "READ")
                {
                    std::vector<uint8_t> q;
                    for (const std::string& x : split(f[2], ',')) q.push_back((uint8_t)atoi(x.c_str()));
                    batch.addRead(f[1], q.data());
                    ++nReads;
                }
                else if (f[0] == "ALN")
                {
                    sx::CandidateAlignment cal;
                    cal.al.pos = atoi(f[2].c_str());
                    sx::cigar_to_apath(f[3].c_str(), cal.al.path);
                    std::map<std::string, bool> cand;
                    const int lead(atoi(f[5].c_str())), trail(atoi(f[6].c_str()));
                    if (f[4] != "-")
                    {
                        int idx(0);
                        for (const std::string& ks : split(f[4], ';'))
                        {
                            const std::vector<std::string> k(split(ks, ':'));
                            const sx::IndelKey key(atoi(k[0].c_str()), (sx::INDEL::index_t)atoi(k[1].c_str()), atoi(k[2].c_str()), k[3] == "-" ? "" : k[3].c_str());
                            cand[k[0] + ":" + k[1] + ":" + k[2] + ":" + (k[3] == "-" ? "" : k[3])] = atoi(k[4].c_str()) != 0;
                            if (idx == lead) cal.leading_indel_key = key;
                            else if (idx == trail) cal.trailing_indel_key = key;
                            else cal.indels.push_back(key);
                            ++idx;
                        }
                    }
                    batch.addCandidateAlignment(regionReadBase + atoi(f[1].c_str()), cal, [&](const sx::IndelKey& key) {
                        return cand[std::to_string(key.pos) + ":" + std::to_string((int)key.type) + ":" + std::to_string(key.deletionLength) + ":" + key.insertSequence];
                    });
                    want.push_back(strtoull(f[7].c_str(), nullptr, 16));
                }
            }
            std::vector<double> got, gotWide;
            batch.scoreCandidateAlignments(ctx, got); // default: the most compact wire formats that fit
            if (!(batch.view().format & SX_FMT_SEG2))
            {
                ++failures;
                std::cerr << "FAIL k1: the batch was expected to fit the compact segment format\n";
            }
            batch.setCompactWireFormats(false);
            batch.scoreCandidateAlignments(ctx, gotWide);
            ++checks;
            if (batch.view().format != 0 || gotWide.size() != got.size() || std::memcmp(gotWide.data(), got.data(), got.size() * sizeof(double)) != 0)
            {
                ++failures;
                std::cerr << "FAIL k1: wide and compact wire formats disagree\n";
            }
            if (got.size() != want.size())
            {
                ++failures;
                std::cerr << "FAIL k1: " << got.size() << " scores, expected " << want.size() << "\n";
            }
            for (size_t i(0); i < got.size() && i < want.size(); ++i)
            {
                uint64_t bits;
                std::memcpy(&bits, &got[i], 8);
                ++checks;
                if (bits != want[i])
                {
                    ++failures;
                    double w;
                    std::memcpy(&w, &want[i], 8);
                    if (failures < 10) std::cerr << "FAIL k1 alignment " << i << ": got " << got[i] << " want " << w << "\n";
                }
            }
        }
        // ---- K6: score_indels through sx::IndelScoreBatch; expected values = the reference's own score_indels on this case
        //      (tests/test_oracle_vs_reference.py pins the oracle, the oracle produced these numbers, the reference harness agreed)
        {
            const double r2i(-9.903487552536127); // ln 5e-5
            std::vector<sx::IndelBufferEntry> window(2);
            window[0].key = sx::IndelKey(1050, sx::INDEL::INDEL, 3, "");
            window[1].key = sx::IndelKey(1052, sx::INDEL::INDEL, 0, "AC");
            for (auto& e : window) e.refToIndelLogProb = e.indelToRefLogProb = r2i;
            sx::IndelScoreBatch ib;
            ib.beginRegion(window);
            auto cal = [](sx::pos_t pos, const char* cigar, std::vector<sx::IndelKey> keys) {
                sx::CandidateAlignment c;
                c.al.pos = pos;
                sx::cigar_to_apath(cigar, c.al.path);
                c.indels = keys;
                return c;
            };
            ib.addRead(100, 99, true, true);
            ib.addCandidateAlignment(cal(1000, "100M", {}));
            ib.addCandidateAlignment(cal(1000, "50M3D50M", {window[0].key}));
            ib.addCandidateAlignment(cal(1000, "52M2I46M", {window[1].key}));
            ib.addRead(60, 60, false, false);
            ib.addCandidateAlignment(cal(1047, "60M", {}));
            ib.addCandidateAlignment(cal(1047, "3M3D57M", {window[0].key}));
            std::vector<sx::IndelScoreBatch::Result> res;
            std::vector<uint32_t> maxAln;
            ib.scoreIndels(ctx, {-20.0, -3.0, -25.0, -4.0, -4.5}, nullptr, res, maxAln);
            auto bitsOf = [](float f) {
                uint32_t u;
                std::memcpy(&u, &f, 4);
                return u;
            };
            ++checks;
            bool ok(res.size() == 3 && maxAln.size() == 2 && maxAln[0] == 1 && maxAln[1] == 3);
            if (ok)
            {
                const sx::ReadPathScores &a(res[0].scores), &b(res[1].scores);
                ok = ok && res[0].read == 0 && res[0].key == window[0].key && !res[0].isSuboverlap && bitsOf(a.ref) == 3243144367u && a.indel == -3.0f &&
                     a.read_pos == 49 && a.distanceFromClosestReadEdge == 49 && a.alt_indel.size() == 1 && a.alt_indel[0].first == window[1].key &&
                     a.alt_indel[0].second == -25.0f && a.nonAmbiguousBasesInRead == 99 && a.read_length == 100 && a.is_tier1_read && a.is_fwd_strand;
                ok = ok && res[1].read == 0 && res[1].key == window[1].key && !res[1].isSuboverlap && bitsOf(b.ref) == 3243144367u && bitsOf(b.indel) == 3243144367u &&
                     b.read_pos == -1 && b.distanceFromClosestReadEdge == 100 && b.alt_indel.size() == 1 && b.alt_indel[0].first == window[0].key &&
                     b.alt_indel[0].second == -3.0f;
                ok = ok && res[2].read == 1 && res[2].key == window[0].key && res[2].isSuboverlap;
            }
            if (!ok)
            {
                ++failures;
                std::cerr << "FAIL k6: IndelScoreBatch::scoreIndels differs from the reference's score_indels on the known-answer case (" << res.size() << " results)\n";
            }
            // a SKIP segment is outside score_indels' domain: the builder refuses it like the reference's assert
            bool threw(false);
            try
            {
                sx::IndelScoreBatch bad;
                bad.beginRegion(window);
                bad.addRead(100, 100, true, true);
                bad.addCandidateAlignment(cal(1000, "50M10N50M", {}));
            }
            catch (const sx::Exception& e)
            {
                threw = (e.code == SX_ERR_UNSUPPORTED);
            }
            ++checks;
            if (!threw)
            {
                ++failures;
                std::cerr << "FAIL k6: a SKIP segment did not raise SX_ERR_UNSUPPORTED\n";
            }
        }
        // ---- error behaviour: a failing call throws, like the reference's blt_exception
        {
            sx::ReadAlignBatch bad;
            bad.beginRegion("ACGTACGTACGTACGT", 0);
            const uint8_t q[4] = {40, 99, 40, 40}; // qphred_cache::qscore_check rejects > 70
            bad.addRead(std::string("ACGT"), q);
            sx::CandidateAlignment cal;
            sx::cigar_to_apath("4M", cal.al.path);
            bad.addCandidateAlignment(0, cal, [](const sx::IndelKey&) { return true; });
            std::vector<double> s;
            bool threw(false);
            try
            {
                bad.scoreCandidateAlignments(ctx, s);
            }
            catch (const sx::Exception& e)
            {
                threw = (e.code == SX_ERR_RANGE);
            }
            ++checks;
            if (!threw)
            {
                ++failures;
                std::cerr << "FAIL: quality 99 did not raise SX_ERR_RANGE\n";
            }
        }
    }
    catch (const std::exception& e)
    {
        std::cerr << "EXCEPTION: " << e.what() << "\n";
        return 3;
    }
    std::cout << "host mirror: " << checks << " checks, " << failures << " failures\n";
    return failures ? 1 : 0;
}
