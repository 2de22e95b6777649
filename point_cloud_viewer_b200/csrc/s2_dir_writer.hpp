// s2_dir_writer.hpp — the host side of the streamed S2 split (s2_stream.inl): appends every batch's per-cell runs to the cells'
// files, the way S2Splitter::write appends each batch to its NodeWriters (src/read_write/s2.rs:73-125), and writes meta.pb last
// (get_meta, :165-173).  Host-only: the CPU tests compile it with g++.
//
// Batches arrive in input order.  The dispatching thread knows every cell's running count before it hands out batch k, so each
// (cell, batch, attribute) run has a fixed file offset: the points of the cell in batches < k times 24 / 3 / 4 bytes.  Any pool
// thread may then write any run, in any order, with pwrite, and the files come out the same.  A cell's files are truncated
// (O_CREAT | O_TRUNC) by the dispatching thread the first time the cell appears, before any of its runs is handed out.  Runs
// open, write and close their file: a cloud may have millions of cells, and no descriptor stays open.
//
// meta.pb is removed by begin(), before any cell file is written, and written by finish() to meta.pb.tmp, then renamed: a call
// that stops early leaves no meta.pb, so the directory does not load.  The first error is recorded and every later run skipped.
#pragma once
#include <fcntl.h>
#include <sys/stat.h>
#include <unistd.h>

#include <algorithm>
#include <cerrno>
#include <condition_variable>
#include <cstdint>
#include <cstring>
#include <deque>
#include <map>
#include <mutex>
#include <string>
#include <thread>
#include <unordered_map>
#include <vector>

#include "s2_disk.hpp"

namespace pcv {

class S2DirWriter {
   public:
    static constexpr int kAttrs = 3;  // xyz, rgb, intensity
    uint64_t bytes_written = 0, file_writes = 0;

    // `has[a]`: the cloud carries attribute a (positions always)
    S2DirWriter(const std::string& dir, int threads, bool has_rgb, bool has_intensity) : dir_(dir) {
        has_[0] = true, has_[1] = has_rgb, has_[2] = has_intensity;
        for (int t = 0; t < std::max(1, threads); ++t) pool_.emplace_back([this] { work(); });
    }
    S2DirWriter(const S2DirWriter&) = delete;
    S2DirWriter& operator=(const S2DirWriter&) = delete;
    ~S2DirWriter() {
        {
            std::lock_guard<std::mutex> l(mu_);
            stop_ = true;
        }
        cv_task_.notify_all();
        for (auto& t : pool_) t.join();
    }

    // Creates the directory if needed ("Ignore errors, maybe directory is already there") and removes its meta.pb.
    bool begin() {
        mkdir(dir_.c_str(), 0777);
        const std::string meta = dir_ + "/meta.pb";
        if (::unlink(meta.c_str()) != 0 && errno != ENOENT) return set_error("cannot remove " + meta);
        return true;
    }

    // Hands out the runs of batch `seq` (seq = 0, 1, ... in input order).  data[a] holds attribute a of the batch's points,
    // cell-contiguous in the order of `ids` (ascending), counts[k] points of cell ids[k]; the buffers must stay valid until
    // wait(seq) returns.  Returns false once an error has been recorded.
    bool submit(uint64_t seq, const uint8_t* const data[kAttrs], const uint64_t* ids, const uint64_t* counts, size_t ncells) {
        static const uint64_t bpp[kAttrs] = {24, 3, 4};
        std::vector<Task> tasks;
        uint64_t off_in[kAttrs] = {0, 0, 0};
        for (size_t k = 0; k < ncells; ++k) {
            if (!ok()) return false;
            const uint64_t id = ids[k], cnt = counts[k];
            auto it = total_.find(id);
            if (it == total_.end()) {  // the cell's first run: truncate its files before any run of it is written
                for (int a = 0; a < kAttrs; ++a) {
                    if (!has_[a]) continue;
                    const std::string path = path_of(id, a);
                    const int fd = ::open(path.c_str(), O_WRONLY | O_CREAT | O_TRUNC, 0666);
                    if (fd < 0 || ::close(fd) != 0) return set_error("cannot write " + path);
                }
                it = total_.emplace(id, 0).first;
            }
            for (int a = 0; a < kAttrs; ++a) {
                if (!has_[a]) continue;
                tasks.push_back(Task{seq, id, a, data[a] + off_in[a], cnt * bpp[a], it->second * bpp[a]});
                off_in[a] += cnt * bpp[a];
                bytes_written += cnt * bpp[a];
                ++file_writes;
            }
            it->second += cnt;
        }
        if (!tasks.empty()) {
            std::lock_guard<std::mutex> l(mu_);
            pending_[seq] += tasks.size();
            for (const Task& t : tasks) queue_.push_back(t);
        }
        cv_task_.notify_all();
        return ok();
    }

    // Blocks until every run of batches <= seq has been written (or skipped after an error).
    void wait(uint64_t seq) {
        std::unique_lock<std::mutex> l(mu_);
        cv_done_.wait(l, [&] { return pending_.empty() || pending_.begin()->first > seq; });
    }
    void wait_all() {
        std::unique_lock<std::mutex> l(mu_);
        cv_done_.wait(l, [&] { return pending_.empty(); });
    }

    // After the last batch: waits for every run, then writes meta.pb (cells in id order) through meta.pb.tmp.
    bool finish(const double bmin[3], const double bmax[3]) {
        wait_all();
        if (!ok()) return false;
        S2MetaData m;
        for (int a = 0; a < 3; ++a) m.bbox_min[a] = bmin[a], m.bbox_max[a] = bmax[a];
        std::vector<std::pair<uint64_t, uint64_t>> cells(total_.begin(), total_.end());
        std::sort(cells.begin(), cells.end());
        for (const auto& c : cells) m.ids.push_back(c.first), m.counts.push_back(c.second);
        m.has_color = has_[1];
        m.has_intensity = has_[2];
        const std::string meta = encode_s2_meta(m), tmp = dir_ + "/meta.pb.tmp", dst = dir_ + "/meta.pb";
        if (!write_whole_file(tmp, meta.data(), meta.size())) return set_error("cannot write " + tmp);
        if (::rename(tmp.c_str(), dst.c_str()) != 0) return set_error("cannot write " + dst);
        return true;
    }

    bool ok() {
        std::lock_guard<std::mutex> l(mu_);
        return err_.empty();
    }
    std::string error() {
        std::lock_guard<std::mutex> l(mu_);
        return err_;
    }
    uint64_t num_cells() const { return total_.size(); }

   private:
    struct Task {
        uint64_t seq, id;
        int attr;
        const uint8_t* p;
        uint64_t len, off;
    };
    std::string dir_;
    bool has_[kAttrs];
    std::unordered_map<uint64_t, uint64_t> total_;  // points per cell so far (dispatching thread only)
    std::mutex mu_;
    std::condition_variable cv_task_, cv_done_;
    std::deque<Task> queue_;
    std::map<uint64_t, uint64_t> pending_;  // batch -> runs not yet finished
    std::string err_;
    bool stop_ = false;
    std::vector<std::thread> pool_;

    std::string path_of(uint64_t id, int a) const {
        static const char* ext[kAttrs] = {".xyz", ".rgb", ".intensity"};
        return dir_ + "/" + s2_to_token(id) + ext[a];
    }
    bool set_error(const std::string& e) {
        std::lock_guard<std::mutex> l(mu_);
        if (err_.empty()) err_ = e;
        return false;
    }
    bool write_run(const Task& t) {
        if (t.len == 0) return true;
        const std::string path = path_of(t.id, t.attr);
        const int fd = ::open(path.c_str(), O_WRONLY);
        if (fd < 0) return set_error("cannot write " + path);
        uint64_t done = 0;
        while (done < t.len) {
            const ssize_t w = ::pwrite(fd, t.p + done, (size_t)(t.len - done), (off_t)(t.off + done));
            if (w <= 0) break;
            done += (uint64_t)w;
        }
        const bool closed = ::close(fd) == 0;
        if (done != t.len || !closed) return set_error("cannot write " + path);
        return true;
    }
    void work() {
        for (;;) {
            Task t;
            bool skip;
            {
                std::unique_lock<std::mutex> l(mu_);
                cv_task_.wait(l, [&] { return stop_ || !queue_.empty(); });
                if (queue_.empty()) return;
                t = queue_.front();
                queue_.pop_front();
                skip = !err_.empty();
            }
            if (!skip) write_run(t);
            std::lock_guard<std::mutex> l(mu_);
            if (--pending_[t.seq] == 0) pending_.erase(t.seq);
            cv_done_.notify_all();
        }
    }
};

}  // namespace pcv
