// plot_html.h — the Chart.js 2 pages of `goleft indexcov` (DESIGN §1.14).  Each chart's config is one JSON object literal,
// written between the markers  /*chart NAME begin*/var cfg_NAME = ... ;/*chart NAME end*/  so that tools can read the data
// back; non-finite numbers are written NaN / Infinity / -Infinity, which JavaScript and Python's json module both read.
#pragma once
#include <math.h>
#include <stdint.h>
#include <string>
#include <vector>

namespace glhtml {

struct Dataset {
    std::string label;
    uint8_t rgb[3] = {0, 0, 0};
    std::vector<double> x, y;
    const char* xfmt = "%.2f";
    const char* yfmt = "%.2f";
    bool line = true;                  // false: points only
    bool stepped = false;              // a stepped line (steppedLine)
    double width = 1;                  // line width, or point radius when !line
};

struct Chart {
    std::string name, xlabel, ylabel;
    std::vector<Dataset> data;
    bool legend = false;
    double ymin = NAN, ymax = NAN;     // fixed y axis ticks when not NaN
    std::string tooltip_js;            // statements run after the chart exists, `chart` bound to it
};

// printf(fmt, v) for a finite v, else NaN / Infinity / -Infinity
std::string num(const char* fmt, double v);
// a JSON string literal
std::string quote(const std::string& s);
// a canvas, the config and the Chart constructor for one chart
std::string chart_html(const Chart& c, int width, int height);
// a whole page: the Chart.js and jQuery scripts, the title, then body
std::string page(const std::string& title, const std::string& body);

// The same markup in pieces, for a page too large to build as one string:
//   page_open(title), then chart_open, then for each dataset "," between datasets, dataset_head(ds), its points
//   {"x":..,"y":..} joined by ",", and "]}", then chart_close, then page_close().
std::string page_open(const std::string& title);
const char* page_close();
std::string chart_open(const Chart& c, int width, int height);
std::string dataset_head(const Dataset& ds);       // ds without its points
std::string chart_close(const Chart& c);

}  // namespace glhtml
