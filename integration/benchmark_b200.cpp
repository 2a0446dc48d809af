// integration/benchmark_b200.cpp -- the reference's accuracy harness (tests/benchmark.cpp:34-150) on this engine, batched.
//
//   usage: benchmark_b200 <model_path> <dataset_dir> <num_images_per_class> [output_file] [batch]
//
// Same contract as the reference tool: <dataset_dir>/<class name>/<image> folders, class names in <dataset_dir>/../classnames.json
// (a JSON array of strings, index = class id), one "file,true class,predicted class" line per image in the output file and a final
// "Top-1 Accuracy: x%" line on stdout.  Differences, all on the fast side of the seam: images are decoded by the reference's own
// load_image_from_file (vit.cpp:108-128, stb_image) and then handed as u8 to vitb200_forward_u8_async in batches (default 256) --
// the bicubic resize + normalisation of vit_image_preprocess and the forward pass run on the GPU, and while batch i is on the GPU the
// host decodes batch i+1 (two pipeline slots).  num_images_per_class is honoured (the reference parses it and then ignores it,
// tests/benchmark.cpp:98-99); 0 = all.  Besides .JPEG the extensions .jpg .jpeg .png .ppm .bmp are accepted.
//
// Built by oracle/Makefile (target cli) against the reference's vit.h / vit.cpp for the loader; needs no nlohmann/json.
#include "vit.h"

#include "vitb200.h"

#include <algorithm>
#include <cstdio>
#include <cstdlib>
#include <filesystem>
#include <fstream>
#include <string>
#include <vector>

namespace fs = std::filesystem;

// JSON array of strings (the only shape classnames.json has); tolerant of whitespace and \" \\ \/ \n \t \uXXXX (kept verbatim) escapes
static std::vector<std::string> read_class_names(const std::string &filename)
{
    std::ifstream f(filename);
    std::vector<std::string> out;
    if (!f)
    {
        fprintf(stderr, "Cannot open file: %s\n", filename.c_str());
        return out;
    }
    std::string s((std::istreambuf_iterator<char>(f)), std::istreambuf_iterator<char>());
    size_t i = 0;
    while (i < s.size() && s[i] != '[') ++i;
    while (i < s.size())
    {
        while (i < s.size() && s[i] != '"' && s[i] != ']') ++i;
        if (i >= s.size() || s[i] == ']') break;
        std::string cur;
        for (++i; i < s.size() && s[i] != '"'; ++i)
        {
            if (s[i] == '\\' && i + 1 < s.size())
            {
                const char c = s[++i];
                if (c == 'n') cur += '\n';
                else if (c == 't') cur += '\t';
                else if (c == 'u') { cur += "\\u"; }
                else cur += c;
            }
            else cur += s[i];
        }
        ++i;
        out.push_back(cur);
    }
    return out;
}

struct Pending
{
    std::vector<image_u8> imgs;
    std::vector<std::string> files, truth;
    std::vector<int32_t> top1;
};

int main(int argc, char **argv)
{
    if (argc < 4)
    {
        fprintf(stderr, "usage: %s <model_path> <dataset_dir> <num_images_per_class> [output_file] [batch]\n", argv[0]);
        return 1;
    }
    const std::string model_path = argv[1], dataset_dir = argv[2];
    const int per_class = atoi(argv[3]);
    const std::string output_file = argc >= 5 ? argv[4] : "predictions.txt";
    const int batch = argc >= 6 ? std::max(1, atoi(argv[5])) : 256;

    const fs::path classnames_path = fs::path(dataset_dir).parent_path() / "classnames.json";
    const std::vector<std::string> CLASS_NAMES = read_class_names(classnames_path.string());

    vitb200_engine *e = nullptr;
    const char *dev = getenv("VITB200_DEVICE");
    if (vitb200_create_from_file(model_path.c_str(), dev ? atoi(dev) : 0, batch, &e) != 0)
    {
        fprintf(stderr, "Failed to load model from %s: %s\n", model_path.c_str(), vitb200_last_error());
        return 1;
    }
    std::ofstream out_file(output_file);
    if (!out_file)
    {
        fprintf(stderr, "Failed to open output file: %s\n", output_file.c_str());
        return 1;
    }

    int total_images = 0, correct_predictions = 0;
    Pending slot[2];
    int cur = 0, in_flight = 0;
    auto flush_results = [&](Pending &p) { // results of a finished batch -> file + counters
        for (size_t i = 0; i < p.files.size(); ++i)
        {
            const int idx = p.top1[i];
            const std::string pred = (idx >= 0 && idx < (int)CLASS_NAMES.size()) ? CLASS_NAMES[idx] : std::to_string(idx);
            if (p.truth[i] == pred) ++correct_predictions;
            ++total_images;
            out_file << p.files[i] << "," << p.truth[i] << "," << pred << std::endl;
        }
        p.imgs.clear(); p.files.clear(); p.truth.clear(); p.top1.clear();
    };
    auto submit = [&](Pending &p) -> bool {
        const int n = (int)p.imgs.size();
        if (n == 0) return true;
        std::vector<const uint8_t *> ptrs(n);
        std::vector<int> nx(n), ny(n);
        for (int i = 0; i < n; ++i) { ptrs[i] = p.imgs[i].data.data(); nx[i] = p.imgs[i].nx; ny[i] = p.imgs[i].ny; }
        p.top1.assign(n, -1);
        // top-1 index only: the head of the reference's sorted `predictions` (vit.cpp:1047-1057)
        if (vitb200_forward_u8_async(e, ptrs.data(), nx.data(), ny.data(), n, /*bilinear*/ 0, nullptr, nullptr, p.top1.data(), nullptr, 1) != 0)
        {
            fprintf(stderr, "Inference failed: %s\n", vitb200_last_error());
            return false;
        }
        return true;
    };

    std::vector<fs::path> classes;
    for (const auto &class_entry : fs::directory_iterator(dataset_dir))
        if (class_entry.is_directory()) classes.push_back(class_entry.path());
    std::sort(classes.begin(), classes.end());
    for (const auto &cdir : classes)
    {
        const std::string class_name = cdir.filename().string();
        std::vector<fs::path> files;
        for (const auto &image_entry : fs::directory_iterator(cdir)) files.push_back(image_entry.path());
        std::sort(files.begin(), files.end());
        int images_processed = 0;
        for (const auto &ipath : files)
        {
            std::string ext = ipath.extension().string();
            std::transform(ext.begin(), ext.end(), ext.begin(), [](unsigned char c) { return (char)tolower(c); });
            if (ext != ".jpeg" && ext != ".jpg" && ext != ".png" && ext != ".ppm" && ext != ".bmp") continue;
            if (per_class > 0 && images_processed >= per_class) break;
            image_u8 img;
            if (!load_image_from_file(ipath.string(), img))
            {
                fprintf(stderr, "Failed to load image from %s\n", ipath.string().c_str());
                continue;
            }
            ++images_processed;
            Pending &p = slot[cur];
            p.imgs.push_back(std::move(img));
            p.files.push_back(ipath.filename().string());
            p.truth.push_back(class_name);
            if ((int)p.imgs.size() == batch)
            {
                if (!submit(p)) return 1;
                // the OTHER slot's batch (submitted one round ago) must be complete before its host buffers are reused: its results are
                // ready once everything submitted so far has drained, which we only wait for when both slots are busy
                ++in_flight;
                cur ^= 1;
                if (in_flight == 2)
                {
                    if (vitb200_sync(e) != 0) { fprintf(stderr, "%s\n", vitb200_last_error()); return 1; }
                    flush_results(slot[cur]);
                    flush_results(slot[cur ^ 1]);
                    in_flight = 0;
                }
            }
        }
    }
    if (!submit(slot[cur])) return 1;
    if (vitb200_sync(e) != 0) { fprintf(stderr, "%s\n", vitb200_last_error()); return 1; }
    flush_results(slot[cur ^ 1]);
    flush_results(slot[cur]);

    const double accuracy = total_images ? static_cast<double>(correct_predictions) / total_images : 0.0;
    printf("Top-1 Accuracy: %g%%\n", accuracy * 100.0);
    vitb200_destroy(e);
    return 0;
}
