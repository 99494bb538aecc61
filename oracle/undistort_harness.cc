/* TEST INFRASTRUCTURE - NOT PRODUCT CODE.
 *
 * Our own driver around the UNMODIFIED reference function mve::image::image_undistort_k2k4<uint8_t>
 * (libs/mve/image_tools.h:1731-1769), the call sfmrecon makes for every view (apps/sfmrecon/sfmrecon.cc:425-437).
 * Built by oracle/undistort.mk into oracle/_ref/undistort_harness with the reference flags:
 *
 *   undistort_harness IN.mvei OUT FLEN K2 K4 [IN.mvei OUT FLEN K2 K4 ...]
 *       Undistorts each 8-bit MVEI image; OUT is an MVEI file, or "-" to discard the result.  FLEN, K2 and K4 are
 *       rounded to float first, as sfmrecon passes CameraInfo's float flen and dist[] (camera.h:161-162).  Every image
 *       is read first, then undistorted one image per thread on all host threads (sfmrecon's OpenMP loop over views);
 *       prints one JSON line with the images, threads and seconds of the undistortion alone.
 */
#include <algorithm>
#include <atomic>
#include <chrono>
#include <cstdio>
#include <cstdlib>
#include <memory>
#include <string>
#include <thread>
#include <vector>

#include "mve/image.h"
#include "mve/image_io.h"
#include "mve/image_tools.h"

int main(int argc, char** argv)
{
    if (argc < 6 || (argc - 1) % 5 != 0) {
        std::fprintf(stderr, "usage: undistort_harness IN OUT FLEN K2 K4 [IN OUT FLEN K2 K4 ...]\n");
        return 2;
    }
    struct Job { mve::ByteImage::Ptr in, out; std::string out_path; double flen, k2, k4; };
    std::vector<Job> jobs;
    for (int a = 1; a < argc; a += 5) {
        Job j;
        j.in = std::dynamic_pointer_cast<mve::ByteImage>(mve::image::load_mvei_file(argv[a]));
        if (j.in == nullptr) { std::fprintf(stderr, "%s: not an 8-bit image\n", argv[a]); return 1; }
        j.out_path = argv[a + 1];
        j.flen = (float)std::atof(argv[a + 2]);
        j.k2 = (float)std::atof(argv[a + 3]);
        j.k4 = (float)std::atof(argv[a + 4]);
        jobs.push_back(j);
    }
    const unsigned n_threads = std::max(1u, std::min<unsigned>(std::thread::hardware_concurrency(), (unsigned)jobs.size()));
    std::atomic<std::size_t> next(0);
    const auto t0 = std::chrono::steady_clock::now();
    std::vector<std::thread> th;
    for (unsigned t = 0; t < n_threads; ++t)
        th.emplace_back([&]() {
            for (std::size_t i; (i = next.fetch_add(1)) < jobs.size();)
                jobs[i].out = mve::image::image_undistort_k2k4<uint8_t>(jobs[i].in, jobs[i].flen, jobs[i].k2, jobs[i].k4);
        });
    for (auto& t : th) t.join();
    const double el = std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
    for (const Job& j : jobs)
        if (j.out_path != "-") mve::image::save_mvei_file(j.out, j.out_path);
    std::printf("{\"images\": %zu, \"threads\": %u, \"seconds\": %.6f}\n", jobs.size(), n_threads, el);
    return 0;
}
