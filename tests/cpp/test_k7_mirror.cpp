// tests/cpp/test_k7_mirror.cpp -- the K7 part of the C++ host mirror on the GPU: sx::AlignmentSearchBatch through the real library
// against the candidate alignments the reference's getCandidateAlignments returned (tests/golden/k7_cases.tsv).  The same check runs
// without a GPU in tests/cpp/test_k7_mirror_cpu.cpp.  Build/run: tests/test_zz_gpu_enumerate.py::test_cpp_host_mirror_k7.
#include "k7_mirror_check.hh"

int main(int argc, char** argv)
{
    if (argc < 2) return 2;
    int checks(0), failures(0);
    try
    {
        sx::Context ctx(0);
        k7_mirror_check(ctx, argv[1], checks, failures);
    }
    catch (const std::exception& e)
    {
        std::cerr << "EXCEPTION: " << e.what() << "\n";
        return 3;
    }
    std::cout << "k7 host mirror: " << checks << " checks, " << failures << " failures\n";
    return failures ? 1 : 0;
}
